"""GPU: the float FFT / MDCT of FFTContext (ff_fft_batch_cuda, ff_mdct_batch_cuda and the slots of ff_fft_init_cuda /
ff_mdct_init_cuda) against the float64 reference of tests/fft64.py, at every size the entry points accept.

Each case runs one batch holding every input class: uniform and Gaussian noise, impulses (every position up to 2^8 inputs, else
0, 1, n/2 - 1, n/2, n - 1 and a random sample), single tones, DC, Nyquist, all-zero, two tones of amplitude 1 and 2^-20, and the
noise times 2^40 and 2^-40.  Per row:
  (a) north star    max |got - want| / max |want| < 1e-6;
  (b) fixed         norm-wise err(got) <= FIXED_K * log2(N) * 2^-24;
      comparative   where oracle/_ref was built, also err(got) <= FACTOR * err(reference) + SLACK_ULP * 2^-24, the reference
                    being the compiled one on the same input (2 points: one float butterfly);
  weak tone         the 2^-20 tone's bin is within WEAK_K * log2(N) * 2^-24 * rms(spectrum) of float64: an absolute bound on
                    that bin, which the north star alone is not (dropping the tone entirely moves the output by 2^-20 < 1e-6
                    of its maximum).  For the IMDCT ops the spectrum is read back by a float64 MDCT of the output;
  exactness         all-zero input gives +-0.0; the 2^+-40 rows are bitwise 2^+-40 times the unscaled rows.
log2(N) is the transform's own size: the FFT's nbits, the MDCT's nbits (not its inner FFT's).

Measured on an H100 80GB HBM3 (the kernels are deterministic, so the numbers do not depend on clocks or power limit): norm-wise
error against float64 in units of 1e-8, largest over input classes, directions or scales, for the GPU and for the compiled
reference on the same inputs.
    FFT         nbits  1    2    3    4    5    6    7    8    9   10   11   12
                GPU   4.3  6.6  5.9  6.6  8.5  8.9 10.5 10.7 11.5 11.9 12.4 14.8
                ref   4.3  6.6  5.3  7.4  9.1  9.1  9.4 11.1 10.8 11.7 11.8 12.3
    imdct_half  nbits  4    5    6    7    8    9   10   11   12   13   14
                GPU   9.8 10.8 11.7 10.9 16.7 14.4 16.1 12.6 13.0 16.5 16.6
                ref   9.7 11.5 11.8 10.9 14.4 12.5 13.9 12.4 12.9 15.6 16.3
    imdct_calc  GPU  10.3 11.4 11.7 11.6 16.7 14.4 16.1 12.6 13.2 16.5 16.6
                ref   9.6  9.9 11.8 12.1 14.4 12.9 13.9 12.6 13.2 15.6 16.3
    mdct_calc   GPU  13.6 14.5 15.4 13.4 21.0 14.8 16.3 15.6 16.6 16.8 19.4
                ref  14.2 14.9 15.1 16.9 20.2 14.1 19.9 16.8 16.1 16.7 20.0
The north star's largest value was 4.1e-7 (imdct at 2^14).  Per row, the largest measured
  err(got) / (log2(N) 2^-24)                   0.72  (FFT 2 points: output rounding alone)  -> FIXED_K = 1.0, margin 1.4
  (err(got) - 2 * 2^-24) / err(reference)      0.75  (imdct 2^13, impulses)                 -> FACTOR = 1.5 with SLACK_ULP = 2,
                                                                                               margin 2.0
  weak-bin error / (log2(N) 2^-24 rms)         0.68  (imdct_calc 2^4)                       -> WEAK_K = 2.0, margin 2.9
With twiddles computed in float instead of double, the FFT's factor rises to 2.3 at 2^5 and 17 at 2^12, the MDCT's to 1.4 at
2^7 and 7.3 at 2^14.
"""
import ctypes as C

import numpy as np
import pytest

import fft64
from oracle import loader
from oracle.loader import ptr

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -24
NORTH_STAR = 1e-6
FACTOR, SLACK_ULP = 1.5, 2.0
FIXED_K = 1.0
WEAK_K = 2.0
WEAK = 2.0 ** -20
SCALES = [1.0, -1.0, 1.0 / 32768, 2.5, -1.0 / 7]
GUARD_BITS, FILL_BITS = 0x7FC0DEAD, 0xFFC0BEEF          # quiet-NaN patterns no transform produces


def _positions(n, rng):
    if n <= 256:
        return list(range(n))
    return sorted({0, 1, n // 2 - 1, n // 2, n - 1} | set(rng.integers(0, n, 8).tolist()))


def _impulses(n, positions):
    a = np.zeros((len(positions), n))
    a[np.arange(len(positions)), positions] = 1
    return a


def _bins(n, rng):
    return sorted({0, 1, n // 2 - 1, n // 2, n - 1} | set(rng.integers(0, n, 3).tolist()))


def _two_bins(n, rng):
    k1 = int(rng.integers(0, n))
    return k1, int((k1 + 1 + rng.integers(0, n - 1)) % n)


def fft_classes(nbits, inverse, rng):
    """[(class, complex rows, weak bin or None)]"""
    n = 1 << nbits
    j = np.arange(n)
    sgn = -1 if inverse else 1                          # the tone that lands in bin k of this direction
    noise = rng.uniform(-1, 1, (2, n)) + 1j * rng.uniform(-1, 1, (2, n))
    k1, k2 = _two_bins(n, rng)
    cls = [("uniform", noise, None),
           ("gauss", rng.standard_normal((2, n)) + 1j * rng.standard_normal((2, n)), None),
           ("impulse", _impulses(n, _positions(n, rng)).astype(complex), None),
           ("tone", np.array([fft64._cis(sgn * k * j, n) for k in _bins(n, rng)]), None),
           ("dc", np.ones((1, n), complex), None),
           ("nyquist", np.array([(-1.0) ** j], complex), None),
           ("zero", np.zeros((1, n), complex), None),
           ("two_tone", (fft64._cis(sgn * k1 * j, n) + WEAK * fft64._cis(sgn * k2 * j, n))[None], k2),
           ("noise*2^40", noise * 2.0 ** 40, None),
           ("noise*2^-40", noise * 2.0 ** -40, None)]
    return [(c, fft64.interleave(r), k) for c, r, k in cls]


def mdct_classes(op, nbits, rng):
    """[(class, real rows, weak bin or None)]"""
    n = 1 << nbits
    nin = fft64.mdct_sizes(op, nbits)[0]
    noise = rng.uniform(-1, 1, (2, nin))
    k1, k2 = _two_bins(n // 2, rng)
    if op == 2:                                         # a tone of the MDCT is one of its basis functions
        basis = lambda k: fft64._cis((2 * np.arange(n) + 1 + n // 2) * (2 * k + 1), 4 * n).real
        tones = np.array([basis(k) for k in _bins(n // 2, rng)])
        two = basis(k1) + WEAK * basis(k2)
    else:                                               # ... of the IMDCT, one coefficient
        tones = None
        two = np.zeros(nin); two[k1], two[k2] = 1, WEAK
    cls = [("uniform", noise, None),
           ("gauss", rng.standard_normal((2, nin)), None),
           ("impulse", _impulses(nin, _positions(nin, rng)), None),
           ("tone", tones, None),
           ("dc", np.ones((1, nin)), None),
           ("nyquist", np.array([(-1.0) ** np.arange(nin)]), None),
           ("zero", np.zeros((1, nin)), None),
           ("two_tone", two[None], k2),
           ("noise*2^40", noise * 2.0 ** 40, None),
           ("noise*2^-40", noise * 2.0 ** -40, None)]
    return [(c, r.astype(np.float32), k) for c, r, k in cls if r is not None]


# ---- calls ----------------------------------------------------------------------------------------------------------
def gpu_fft(gpu, nbits, inverse, zf):
    from libav_b200 import device
    d = device.DevBuf.from_numpy(zf)
    gpu.check(gpu.lib.ff_fft_batch_cuda(nbits, inverse, d.ptr, zf.shape[0], None), "ff_fft_batch_cuda")
    device.sync()
    return d.download(np.float32, zf.shape)


def gpu_mdct(gpu, op, nbits, scale, x):
    from libav_b200 import device
    T, nout = x.shape[0], fft64.mdct_sizes(op, nbits)[1]
    d_in, d_out = device.DevBuf.from_numpy(x), device.DevBuf(4 * T * nout)
    gpu.check(gpu.lib.ff_mdct_batch_cuda(op, nbits, scale, d_out.ptr, d_in.ptr, T, None), "ff_mdct_batch_cuda")
    device.sync()
    return d_out.download(np.float32, (T, nout))


def ref_fft(ref, nbits, inverse, zf):
    """the compiled reference's float result per row (its ff_fft_init starts at 4 points; 2 points is one float butterfly)"""
    if nbits == 1:
        z = fft64.cplx(zf).astype(np.complex64)
        return fft64.interleave(np.stack([z[:, 0] + z[:, 1], z[:, 0] - z[:, 1]], axis=1))
    out = zf.copy()
    for t in range(out.shape[0]):
        ref.fft(nbits, inverse, ptr(out[t]))
    return out


def ref_mdct(ref, op, nbits, scale, x):
    out = np.zeros((x.shape[0], fft64.mdct_sizes(op, nbits)[1]), np.float32)
    for t in range(x.shape[0]):
        getattr(ref, fft64.OPS[op])(nbits, scale, ptr(out[t]), ptr(x[t].copy()))
    return out


def full_imdct(half, nbits):
    """imdct_calc's output rebuilt from imdct_half's by the mirror of mdct_template.c:141-144"""
    n4 = 1 << (nbits - 2)
    return np.concatenate([-half[..., :n4][..., ::-1], half, half[..., n4:][..., ::-1]], axis=-1)


def spectrum(kind, nbits, out):
    """where a two-tone input's weak tone shows: the output itself, or for the IMDCT ops a float64 MDCT of it"""
    if kind in ("fft", 2):
        return out
    return fft64.mdct_calc(full_imdct(out, nbits) if kind == 0 else out, nbits, 1.0)


# ---- checks ---------------------------------------------------------------------------------------------------------
def check_batch(label, kind, nbits, classes, got, want, ref, to_vals):
    """got / ref: float32 outputs of the whole batch; want: float64 (complex for the FFT); to_vals maps float rows to values"""
    assert np.isfinite(got).all(), label
    g, r = to_vals(got), to_vals(ref) if ref is not None else None
    e_g = fft64.err(g, want)
    e_r = fft64.err(r, want) if r is not None else None
    ns = fft64.max_rel(g, want)
    row, rows, checks, stats = 0, {}, [], {}
    for c, rws, weak in classes:
        sl = slice(row, row + rws.shape[0])
        row += rws.shape[0]
        rows[c] = sl
        stat = {"gpu": float(e_g[sl].max()), "north_star": float(ns[sl].max()),
                "fixed_k": float(e_g[sl].max() / (nbits * ULP))}
        checks += [(c, "north star", ns[sl] < NORTH_STAR), (c, "fixed bound", e_g[sl] <= FIXED_K * nbits * ULP)]
        if e_r is not None:
            stat["ref"] = float(e_r[sl].max())
            stat["factor"] = float(((e_g[sl] - SLACK_ULP * ULP) / np.maximum(e_r[sl], 1e-30)).max())
            checks.append((c, "against the reference", e_g[sl] <= FACTOR * e_r[sl] + SLACK_ULP * ULP))
        if weak is not None:
            sg, sw = spectrum(kind, nbits, g[sl]), spectrum(kind, nbits, want[sl])
            unit = nbits * ULP * np.linalg.norm(sw, axis=-1) / np.sqrt(sw.shape[-1])
            stat["weak_k"] = float((np.abs(sg[:, weak] - sw[:, weak]) / unit).max())
            checks += [(c, "the bound sees the weak tone", WEAK_K * unit < 0.5 * np.abs(sw[:, weak])),
                       (c, "weak tone", np.abs(sg[:, weak] - sw[:, weak]) <= WEAK_K * unit)]
        if c == "zero":
            checks.append((c, "+-0.0 out", got[sl] == 0))
        stats[c] = stat
    for c, what, ok in checks:
        assert np.all(ok), (label, c, what, stats[c])
    # scaling by a power of two commutes with the transform exactly: no row here over- or underflows
    base = got[rows["uniform"]]
    assert np.array_equal(got[rows["noise*2^40"]], base * np.float32(2.0 ** 40)), label
    assert np.array_equal(got[rows["noise*2^-40"]], base * np.float32(2.0 ** -40)), label


@pytest.mark.parametrize("nbits", range(1, 13))
@pytest.mark.parametrize("inverse", [0, 1])
def test_fft_batch_accuracy(gpu, nbits, inverse):
    rng = np.random.default_rng(100 + 2 * nbits + inverse)
    classes = fft_classes(nbits, inverse, rng)
    zf = np.concatenate([r for _, r, _ in classes])
    got = gpu_fft(gpu, nbits, inverse, zf)
    ref = loader.ref()
    check_batch("fft nbits %d inverse %d" % (nbits, inverse), "fft", nbits, classes, got, fft64.fft(fft64.cplx(zf), inverse),
                ref_fft(ref, nbits, inverse, zf) if ref else None, fft64.cplx)
    row = 0
    for c, r, _ in classes:                             # tones: all energy in their own bin
        if c == "tone":
            assert np.array_equal(np.abs(fft64.cplx(got[row:row + len(r)])).argmax(axis=-1),
                                  np.abs(fft64.fft(fft64.cplx(r), inverse)).argmax(axis=-1))
        row += len(r)


@pytest.mark.parametrize("nbits", range(1, 13))
@pytest.mark.parametrize("inverse", [0, 1])
def test_fft_of_impulse_at_one_is_the_rounded_twiddles(gpu, nbits, inverse):
    """An impulse at index 1 reaches the last radix-2 stage as ones in the upper half and zeros in the lower half, so output k is
    exactly +-1 times that stage's twiddle k mod n/2.  Each component must be the float rounding of a double-precision
    exp(-+2 pi i k / n): within half a float ulp of the exact value, plus double rounding (cos(pi / 2) is 6e-17 in double, not
    0).  Twiddles computed in float miss by ulps, a wrong index by far more."""
    n = 1 << nbits
    z = fft64.interleave(_impulses(n, [1]))
    got = fft64.cplx(gpu_fft(gpu, nbits, inverse, z))[0]
    k = np.arange(n)
    want = np.where(k < n // 2, 1, -1) * fft64._cis((1 if inverse else -1) * (k % max(n // 2, 1)), n)
    for part in (np.real, np.imag):
        tol = np.spacing(np.abs(part(want)).astype(np.float32)).astype(np.float64) / 2 + 2.0 ** -50
        bad = np.flatnonzero(np.abs(part(got) - part(want)) > tol)
        assert bad.size == 0, (part.__name__, bad[:8], got[bad[:8]], want[bad[:8]])


MDCT_CASES = [(op, nbits, scale) for nbits in range(4, 15) for op in range(3) for scale in SCALES]


@pytest.mark.parametrize("op,nbits,scale", MDCT_CASES, ids=["%s-%d-s%g" % (fft64.OPS[o], b, s) for o, b, s in MDCT_CASES])
def test_mdct_batch_accuracy(gpu, op, nbits, scale):
    rng = np.random.default_rng(1000 + 3 * nbits + op)
    classes = mdct_classes(op, nbits, rng)
    x = np.concatenate([r for _, r, _ in classes])
    got = gpu_mdct(gpu, op, nbits, scale, x)
    ref = loader.ref()
    check_batch("%s nbits %d scale %g" % (fft64.OPS[op], nbits, scale), op, nbits, classes, got, fft64.mdct_op(op, x, nbits, scale),
                ref_mdct(ref, op, nbits, scale, x) if ref else None, lambda a: a)


# ---- batch invariance -----------------------------------------------------------------------------------------------
INVARIANCE = [("fft", 0, 4, 0.0), ("fft", 1, 4, 0.0), ("mdct", 0, 5, -1.0), ("mdct", 1, 5, 2.5), ("mdct", 2, 5, 1.0 / 32768)]


def _run(gpu, what, x):
    kind, a, nbits, scale = what
    return gpu_fft(gpu, nbits, a, x) if kind == "fft" else gpu_mdct(gpu, a, nbits, scale, x)


@pytest.mark.parametrize("what", INVARIANCE, ids=["%s-%d-%d" % w[:3] for w in INVARIANCE])
@pytest.mark.parametrize("T", [1, 37, 65537])
def test_batch_invariance(gpu, what, T):
    """transform t of a batch is bitwise the same input transformed alone, whatever the batch size"""
    kind, a, nbits, _ = what
    nin = 2 << nbits if kind == "fft" else fft64.mdct_sizes(a, nbits)[0]
    base = np.random.default_rng(T).standard_normal((min(T, 37), nin)).astype(np.float32)
    alone = np.concatenate([_run(gpu, what, base[i:i + 1]) for i in range(base.shape[0])])
    got = _run(gpu, what, base[np.arange(T) % base.shape[0]])
    assert np.array_equal(got, alone[np.arange(T) % base.shape[0]])


def test_bench_shape(gpu):
    """bench.py's fft workload: 32768 forward 1024-point transforms in one call, a sample checked against float64, some bitwise
    against the same input transformed alone"""
    nbits, T = 10, 32768
    rng = np.random.default_rng(7)
    zf = rng.standard_normal((T, 2 << nbits), dtype=np.float32)
    got = gpu_fft(gpu, nbits, 0, zf)
    sample = np.unique(np.concatenate([[0, 1, T // 2, T - 1], rng.integers(0, T, 60)]))
    want = fft64.fft(fft64.cplx(zf[sample]), 0)
    g = fft64.cplx(got[sample])
    assert (fft64.max_rel(g, want) < NORTH_STAR).all()
    assert (fft64.err(g, want) <= FIXED_K * nbits * ULP).all()
    ref = loader.ref()
    if ref:
        assert (fft64.err(g, want) <= FACTOR * fft64.err(fft64.cplx(ref_fft(ref, nbits, 0, zf[sample])), want) + SLACK_ULP * ULP).all()
    for t in sample[::8]:
        assert np.array_equal(gpu_fft(gpu, nbits, 0, zf[t:t + 1]), got[t:t + 1]), t


# ---- boundaries -----------------------------------------------------------------------------------------------------
class Guarded:
    """a device buffer of `n` floats between G guard floats on each side, all set from the host"""
    G = 64

    def __init__(self, data_bits):
        from libav_b200 import device
        self.n = data_bits.size
        g = np.full(self.G, GUARD_BITS, np.uint32)
        self.host = np.concatenate([g, data_bits.view(np.uint32).ravel(), g])
        self.buf = device.DevBuf.from_numpy(self.host)
        self.ptr = self.buf.ptr + 4 * self.G

    def read(self):
        """(guards before and after, data) as uint32"""
        a = self.buf.download(np.uint32, self.host.shape)
        return np.concatenate([a[:self.G], a[-self.G:]]), a[self.G:-self.G]

    def guards_intact(self):
        return (self.read()[0] == GUARD_BITS).all()


@pytest.mark.parametrize("nbits", [1, 5, 12])
def test_fft_writes_inside_its_buffer(gpu, nbits):
    T = 3
    zf = np.random.default_rng(nbits).uniform(-1, 1, (T, 2 << nbits)).astype(np.float32)
    b = Guarded(zf)
    gpu.check(gpu.lib.ff_fft_batch_cuda(nbits, 1, b.ptr, T, None), "ff_fft_batch_cuda")
    from libav_b200 import device
    device.sync()
    guards, data = b.read()
    assert (guards == GUARD_BITS).all()
    assert np.array_equal(data.view(np.float32).reshape(T, -1), gpu_fft(gpu, nbits, 1, zf))


@pytest.mark.parametrize("op", range(3))
@pytest.mark.parametrize("nbits", [4, 9, 14])
def test_mdct_writes_inside_its_buffer(gpu, op, nbits):
    """guards on both buffers unchanged, every one of the T * nout output floats written, the input bitwise unchanged"""
    from libav_b200 import device
    T = 3
    nin, nout = fft64.mdct_sizes(op, nbits)
    x = np.random.default_rng(nbits + op).uniform(-1, 1, (T, nin)).astype(np.float32)
    bi, bo = Guarded(x), Guarded(np.full(T * nout, FILL_BITS, np.uint32))
    gpu.check(gpu.lib.ff_mdct_batch_cuda(op, nbits, -1.0, bo.ptr, bi.ptr, T, None), "ff_mdct_batch_cuda")
    device.sync()
    (gi, di), (go, do) = bi.read(), bo.read()
    assert (gi == GUARD_BITS).all() and (go == GUARD_BITS).all()
    assert np.array_equal(di, x.view(np.uint32).ravel())
    assert not (do == FILL_BITS).any()
    assert np.array_equal(do.view(np.float32).reshape(T, nout), gpu_mdct(gpu, op, nbits, -1.0, x))


def test_on_a_stream(gpu):
    """h2d, transform and d2h queued on one stream, then that stream synchronised: the default stream's results"""
    from libav_b200 import device
    lib = gpu.lib
    st = lib.avb200_stream_create()
    assert st, gpu.last_error()
    try:
        rng = np.random.default_rng(11)
        for what in [("fft", 0, 10, 0.0), ("fft", 1, 12, 0.0)] + [("mdct", op, 11, -1.0 / 7) for op in range(3)]:
            kind, a, nbits, scale = what
            T = 257
            nin, nout = (2 << nbits, 2 << nbits) if kind == "fft" else fft64.mdct_sizes(a, nbits)
            x = rng.standard_normal((T, nin)).astype(np.float32)
            out = np.zeros((T, nout), np.float32)
            d_in = device.DevBuf(x.nbytes)
            d_out = d_in if kind == "fft" else device.DevBuf(out.nbytes)
            gpu.check(lib.avb200_memcpy_h2d(d_in.ptr, ptr(x), x.nbytes, st), "h2d")
            if kind == "fft":
                gpu.check(lib.ff_fft_batch_cuda(nbits, a, d_in.ptr, T, st), "fft")
            else:
                gpu.check(lib.ff_mdct_batch_cuda(a, nbits, scale, d_out.ptr, d_in.ptr, T, st), "mdct")
            gpu.check(lib.avb200_memcpy_d2h(ptr(out), d_out.ptr, out.nbytes, st), "d2h")
            gpu.check(lib.avb200_stream_sync(st), "stream sync")
            assert np.array_equal(out, _run(gpu, what, x)), what
    finally:
        lib.avb200_stream_destroy(st)
    assert gpu.last_error() == ""


REFUSALS = [("fft", 0, 0, 0.0), ("fft", 0, 13, 0.0), ("fft", 1, -1, 0.0), ("mdct", 0, 3, 1.0), ("mdct", 1, 15, 1.0),
            ("mdct", -1, 8, 1.0), ("mdct", 3, 8, 1.0)]


@pytest.mark.parametrize("what", REFUSALS, ids=["%s-op%d-nbits%d" % w[:3] for w in REFUSALS])
def test_refusal_leaves_buffers_alone(gpu, what):
    from libav_b200 import device
    kind, a, nbits, scale = what
    lib = gpu.lib
    lib.avb200_clear_error()
    x = np.random.default_rng(3).uniform(-1, 1, 2 * 4096).astype(np.float32)       # more than any accepted size reads
    bi, bo = Guarded(x), Guarded(np.full(2 * 4096, FILL_BITS, np.uint32))
    rc = lib.ff_fft_batch_cuda(nbits, a, bi.ptr, 2, None) if kind == "fft" else lib.ff_mdct_batch_cuda(a, nbits, scale, bo.ptr, bi.ptr, 2, None)
    assert rc == -1
    assert gpu.last_error() != ""
    lib.avb200_clear_error()
    device.sync()
    assert np.array_equal(bi.read()[1], x.view(np.uint32)) and bi.guards_intact()
    assert (bo.read()[1] == FILL_BITS).all() and bo.guards_intact()


def test_zero_transforms(gpu):
    from libav_b200 import device
    lib = gpu.lib
    x = np.random.default_rng(4).uniform(-1, 1, 4096).astype(np.float32)
    bi, bo = Guarded(x), Guarded(np.full(4096, FILL_BITS, np.uint32))
    assert lib.ff_fft_batch_cuda(10, 0, bi.ptr, 0, None) == 0
    for op in range(3):
        assert lib.ff_mdct_batch_cuda(op, 10, 1.0, bo.ptr, bi.ptr, 0, None) == 0
    device.sync()
    assert np.array_equal(bi.read()[1], x.view(np.uint32)) and (bo.read()[1] == FILL_BITS).all()
    assert gpu.last_error() == ""


# ---- slots on the reference's own contexts --------------------------------------------------------------------------
def _ctx(refo, nbits, inverse, mdct, scale):
    from libav_b200 import tables
    lib = refo.lib
    lib.ref_fft_ctx_new.restype = C.c_void_p
    lib.ref_fft_ctx_new.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double]
    lib.ref_fft_ctx_free.argtypes = [C.c_void_p, C.c_int]
    p = lib.ref_fft_ctx_new(nbits, inverse, mdct, scale)
    assert p
    return p, C.cast(p, C.POINTER(tables.FFTContext))


def _fptr(f):
    return C.cast(f, C.c_void_p).value


@pytest.mark.parametrize("nbits", range(2, 17))
@pytest.mark.parametrize("inverse", [0, 1])
def test_fft_slot(gpu, refo, nbits, inverse):
    """fft_permute (the reference's) + fft_calc (CUDA from 2^2 to 2^12 points; above, the context keeps its C fft_calc)"""
    p, ctx = _ctx(refo, nbits, inverse, 0, 1.0)
    try:
        c_calc = _fptr(ctx.contents.fft_calc)
        rng = np.random.default_rng(nbits)
        n = 1 << nbits
        rows = [fft64.interleave(r) for r in (rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n), *_impulses(n, [1, n - 1]),
                                               fft64._cis((-1 if inverse else 1) * 3 * np.arange(n), n))]
        want_c = []
        for z in rows:
            a = z.copy()
            ctx.contents.fft_permute(ctx, ptr(a)); ctx.contents.fft_calc(ctx, ptr(a))
            want_c.append(a)
        gpu.lib.ff_fft_init_cuda(ctx)
        assert (_fptr(ctx.contents.fft_calc) == c_calc) == (nbits > 12)
        for z, r in zip(rows, want_c):
            a = z.copy()
            ctx.contents.fft_permute(ctx, ptr(a)); ctx.contents.fft_calc(ctx, ptr(a))
            want = fft64.fft(fft64.cplx(z), inverse)
            assert fft64.max_rel(fft64.cplx(a), want) < NORTH_STAR
            assert fft64.err(fft64.cplx(a), want) <= FACTOR * fft64.err(fft64.cplx(r), want) + SLACK_ULP * ULP
            if nbits <= 12:                             # the revtab gather feeds the same kernel as the natural-order batch call
                assert np.array_equal(a, gpu_fft(gpu, nbits, inverse, z[None])[0])
    finally:
        refo.lib.ref_fft_ctx_free(p, 0)
    assert gpu.last_error() == ""


@pytest.mark.parametrize("nbits", range(4, 16))
@pytest.mark.parametrize("scale", [1.0, -1.0 / 7])
def test_mdct_slots(gpu, refo, nbits, scale):
    """imdct_calc / imdct_half on an inverse context, mdct_calc / mdct_calcw on a forward one (CUDA from 2^4 to 2^14; above,
    the context keeps its C slots)"""
    from libav_b200 import tables
    n = 1 << nbits
    rng = np.random.default_rng(nbits)
    for inverse, fields in ((1, ("imdct_half", "imdct_calc")), (0, ("mdct_calc", "mdct_calcw"))):
        p, ctx = _ctx(refo, nbits, inverse, 1, scale)
        try:
            slot = lambda f: tables._mdctf(ctx.contents.mdct_calcw) if f == "mdct_calcw" else getattr(ctx.contents, f)
            before = {f: _fptr(slot(f)) for f in fields}
            x = rng.uniform(-1, 1, n if inverse == 0 else n // 2).astype(np.float32)
            want_c = {}
            for f in fields:
                out = np.zeros(n, np.float32)
                slot(f)(ctx, out.ctypes.data_as(C.POINTER(C.c_float)), x.ctypes.data_as(C.POINTER(C.c_float)))
                want_c[f] = out
            gpu.lib.ff_mdct_init_cuda(ctx)
            for f in fields:
                assert (_fptr(slot(f)) == before[f]) == (nbits > 14), f
                op = {"imdct_half": 0, "imdct_calc": 1, "mdct_calc": 2, "mdct_calcw": 2}[f]
                nout = fft64.mdct_sizes(op, nbits)[1]
                out = np.full(n, np.nan, np.float32)
                slot(f)(ctx, out.ctypes.data_as(C.POINTER(C.c_float)), x.ctypes.data_as(C.POINTER(C.c_float)))
                assert np.isnan(out[nout:]).all(), f
                want = fft64.mdct_op(op, x, nbits, scale)
                assert fft64.max_rel(out[:nout], want) < NORTH_STAR, f
                assert fft64.err(out[:nout], want) <= FACTOR * fft64.err(want_c[f][:nout], want) + SLACK_ULP * ULP, f
                if nbits <= 14:     # the context's tcos / tsin (ff_mdct_init) equal the rotation tables the batch call builds
                    assert np.array_equal(out[:nout], gpu_mdct(gpu, op, nbits, scale, x[None])[0]), f
        finally:
            refo.lib.ref_fft_ctx_free(p, 1)
    assert gpu.last_error() == ""
