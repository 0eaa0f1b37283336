"""The batched H.264 intra reconstruction against the reference on the pictures of tests/h264_intra_cases.py: slices that start anywhere and
constrained_intra_pred, so availability inside the picture comes from the masks alone; every prediction mode after the decoder's
substitutions; int16 wrap-around and every dispatch rule of the residual.  Every case compares the pixels and the whole coefficient arena
(elements 576..767 and the stride padding are poisoned and must come back unchanged); in decoder layout every guard and padding byte too.

What h264_intra_kernel (libav_b200/csrc/h264intra.cu) does differently by its arguments: coeff_stride % 8 == 0 with a 16-byte aligned arena
fetches and writes back coefficient rows in 16-byte pieces, anything else in 4-byte pieces (stride 772, an arena at +4 bytes).  Arguments it
cannot take are refused before anything is queued: planes or pitches off 4-byte alignment, mbs / nnzc / coeffs off 4-byte alignment, an odd
coeff_stride or one below 768, NULL pointers; ff_h264_flush_pictures_cuda refuses the same before its first stage.  Rows are handed out by
an atomic ticket, so a batch with more rows than the GPU holds at once must still finish."""
import ctypes as C

import numpy as np
import pytest

from libav_b200 import synth
import h264_edge_cases as ec
import h264_hbd_util as hh
import h264_intra_cases as ic
import h264_util as hu
from test_gpu_h264_edges import Placed, _dev, flush_batch

pytestmark = pytest.mark.gpu
TIGHT = ec.Layout("tight", 0, 0)
KEYS = [(w, h, s, c) for (w, h) in ic.SIZES for (s, c) in ic.VARIANTS]
key_id = lambda k: "%dx%d-slices%d-cip%d" % k


@pytest.fixture(scope="module")
def cases(checker):
    """the matrix, each picture with what the checker makes of it: (planes, coefficient arena)"""
    out = ic.matrix_cases()
    for (mb_w, mb_h, _, _), c in out.items():
        want, co = [p.copy() for p in c["planes"]], c["coeffs"].copy()
        hu.oracle_intra(checker, c["rec"], co, c["nnzc"], mb_w, mb_h, *want)
        c["want"] = (want, co)
    return out


def arena(co, stride, shift):
    """the coefficient rows at `stride` elements, `shift` bytes into an allocation of 0x5A bytes"""
    n = co.shape[0]
    buf = np.full(shift + co.itemsize * n * stride + 16, 0x5A, np.uint8)
    buf[shift:shift + co.itemsize * n * stride].view(co.dtype).reshape(n, stride)[:, :768] = co
    return buf


def run_intra(gpu, rec, co, nnzc, mb_w, mb_h, P, planes, lay, stride=768, shift=0):
    """ff_h264_intra_mb_batch_cuda on planes placed by `lay`: returns the placed pictures and the arena's bytes"""
    from libav_b200 import device
    d, buf = Placed(lay, planes), arena(co, stride, shift)
    d_rec, d_nz, d_co, prog = _dev(rec), _dev(nnzc), _dev(buf), device.DevBuf(4 * mb_h * P)
    gpu.check(gpu.lib.ff_h264_intra_mb_batch_cuda(d_rec.ptr, mb_w, mb_h, P, d_co.ptr + shift, stride, d_nz.ptr, *d.ptrs, d.ls[0], d.ls[1],
                                                  prog.ptr, None))
    device.sync()
    return d, d_co.download(np.uint8, buf.shape)


def check_arena(got, want_co, stride, shift):
    want = arena(want_co, stride, shift)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5].tolist()


@pytest.mark.parametrize("lay", [TIGHT, ec.PAD4], ids=repr)
@pytest.mark.parametrize("key", KEYS, ids=key_id)
def test_availability_matrix(gpu, cases, key, lay):
    mb_w, mb_h = key[:2]
    c = cases[key]
    d, got = run_intra(gpu, c["rec"], c["coeffs"], c["nnzc"], mb_w, mb_h, 1, c["planes"], lay)
    d.check(c["want"][0], key)
    check_arena(got, c["want"][1], 768, 0)


@pytest.mark.parametrize("stride,shift", [(768, 0), (776, 0), (772, 0), (768, 4)])
def test_arena_stride_and_alignment(gpu, cases, stride, shift):
    """768 / 776: 16-byte rows; 772 and an arena at +4 bytes: 4-byte rows.  The same pixels and coefficients either way."""
    c = cases[11, 7, True, True]
    d, got = run_intra(gpu, c["rec"], c["coeffs"], c["nnzc"], 11, 7, 1, c["planes"], ec.PAD4, stride, shift)
    d.check(c["want"][0])
    check_arena(got, c["want"][1], stride, shift)


# ---- refusals: -1 with a message, nothing queued, no buffer changed ----
class Refusal:
    """the buffers of one 8-bit call, each inside a poisoned allocation that lets a pointer be moved off alignment"""

    def __init__(self, c, mb_w, mb_h, lay=ec.PAD4):
        from libav_b200 import device
        self.c, self.mb_w, self.mb_h = c, mb_w, mb_h
        self.d = Placed(lay, c["planes"])
        self.host = dict(rec=np.pad(c["rec"].view(np.uint8), (0, 8), constant_values=0x5A),
                         nz=np.pad(c["nnzc"].reshape(-1), (0, 8), constant_values=0x5A), co=arena(c["coeffs"], 768, 0),
                         prog=np.full(4 * mb_h, 0xEE, np.uint8))
        self.dev = {k: _dev(v) for k, v in self.host.items()}
        self.device = device

    def call(self, gpu, stride=768, rec=0, nz=0, co=0, null=None):
        p = {k: v.ptr for k, v in self.dev.items()}
        planes = dict(zip(("luma", "cb", "cr"), self.d.ptrs))
        args = dict(mbs=p["rec"] + rec, coeffs=p["co"] + co, nnzc=p["nz"] + nz, progress=p["prog"], **planes)
        if null:
            args[null] = None
        return gpu.lib.ff_h264_intra_mb_batch_cuda(args["mbs"], self.mb_w, self.mb_h, 1, args["coeffs"], stride, args["nnzc"], args["luma"],
                                                    args["cb"], args["cr"], self.d.ls[0], self.d.ls[1], args["progress"], None)

    def unchanged(self):
        self.device.sync()
        self.d.check(self.c["planes"], "refused")
        for k, v in self.host.items():
            assert np.array_equal(self.dev[k].download(np.uint8, v.shape), v), k


def refused(gpu, rc, what):
    assert rc == -1
    msg = gpu.last_error()
    gpu.lib.avb200_clear_error()
    assert what in msg, msg


@pytest.mark.parametrize("lay", [ec.PAD2, ec.SHIFT1, ec.SHIFT2, ec.ODD_UV, ec.ODD_CB], ids=repr)
def test_refuses_unaligned_planes(gpu, cases, lay):
    r = Refusal(cases[3, 2, True, True], 3, 2, lay)
    refused(gpu, r.call(gpu), "4-byte aligned")
    r.unchanged()


@pytest.mark.parametrize("args,what", [(dict(stride=576), "at least 768"), (dict(stride=767), "coeff_stride even"),
                                       (dict(stride=769), "coeff_stride even"), (dict(co=2), "4-byte aligned"),
                                       (dict(rec=2), "4-byte aligned"), (dict(nz=2), "4-byte aligned")] +
                         [(dict(null=k), "NULL") for k in ("mbs", "coeffs", "nnzc", "luma", "cb", "cr", "progress")],
                         ids=lambda v: ",".join("%s=%s" % kv for kv in v.items()) if isinstance(v, dict) else v)
def test_refuses_arguments_the_kernel_cannot_take(gpu, cases, args, what):
    r = Refusal(cases[3, 2, True, True], 3, 2)
    refused(gpu, r.call(gpu, **args), what)
    r.unchanged()


@pytest.mark.parametrize("bits,c422,shift", [(9, 0, 2), (10, 0, 2), (9, 1, 2), (10, 1, 2), (8, 1, 1)])
def test_hbd_refuses_unaligned_arena(gpu, bits, c422, shift):
    """int32 coefficients at 9 / 10 bit, int16 at 8-bit 4:2:2: an arena off that alignment is refused"""
    from libav_b200 import device
    mb_w, mb_h = 3, 2
    c = ic.intra_case(mb_w, mb_h, 5, True, True, bits, c422)
    y, cb, cr = c["planes"]
    buf = arena(c["coeffs"], 768, 0)
    d = [_dev(v) for v in (c["rec"], c["nnzc"], buf, y, cb, cr)]
    fn = gpu.lib.ff_h264_intra_mb_batch_422_cuda if c422 else gpu.lib.ff_h264_intra_mb_batch_hbd_cuda
    refused(gpu, fn(bits, d[0].ptr, mb_w, mb_h, 1, d[2].ptr + shift, 768, d[1].ptr, d[3].ptr, d[4].ptr, d[5].ptr, y.strides[0], cb.strides[0],
                    None), "aligned to its coefficient type")
    device.sync()
    for dv, v in zip(d[2:], (buf, y, cb, cr)):
        assert np.array_equal(dv.download(v.dtype, v.shape), v)


# ---- stacked and oversized batches ----
def stacked(gpu, checker, pics, mb_w, mb_h, lay):
    """pictures with their own slices and constraints in one call; each against its own checker run"""
    want, want_co = [], []
    for c in pics:
        w, co = [p.copy() for p in c["planes"]], c["coeffs"].copy()
        hu.oracle_intra(checker, c["rec"], co, c["nnzc"], mb_w, mb_h, *w)
        want.append(w)
        want_co.append(co)
    cat = lambda k: np.concatenate([c[k] for c in pics])
    d, got = run_intra(gpu, cat("rec"), cat("coeffs"), cat("nnzc"), mb_w, mb_h, len(pics),
                       [np.concatenate([c["planes"][i] for c in pics]) for i in range(3)], lay)
    d.check([np.concatenate([w[i] for w in want]) for i in range(3)])
    check_arena(got, np.concatenate(want_co), 768, 0)


def test_stacked_pictures_with_their_own_slices(gpu, checker):
    stacked(gpu, checker, [ic.intra_case(11, 7, 90 + k, s, c) for k, (s, c) in enumerate(ic.VARIANTS * 2)], 11, 7, ec.PAD4)


def sm_count():
    cu = C.CDLL("libcuda.so.1")
    dev, n = C.c_int(), C.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetAttribute(C.byref(n), 16, dev) == 0               # CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT
    return n.value


def test_more_rows_than_the_gpu_holds_at_once(gpu, checker):
    """a 32-thread CTA per row with ~5 KB of shared memory: 32 CTAs per SM are resident, so 32 x SMs rows run at once; the rest must wait
    for rows to finish and still be served in ticket order"""
    mb_w, mb_h = 2, 68
    P = 32 * sm_count() // mb_h + 1
    assert P * mb_h > 32 * sm_count()
    stacked(gpu, checker, [ic.intra_case(mb_w, mb_h, 200 + k, *ic.VARIANTS[k % 4]) for k in range(P)], mb_w, mb_h, TIGHT)


# ---- the other two entry points: the same records at 9 / 10 bit and 4:2:2 ----
@pytest.mark.parametrize("bits,c422", [(9, 0), (10, 0), (8, 1), (9, 1), (10, 1)])
@pytest.mark.parametrize("mb_w,mb_h", [(3, 2), (11, 7)])
def test_hbd_and_422_entry_points(gpu, checker, bits, c422, mb_w, mb_h):
    """every availability variant stacked in one call; int16 wrap-around kinds at 8 bit, int32 up to +-2^20 at 9 / 10"""
    from libav_b200 import device
    pics = [ic.intra_case(mb_w, mb_h, 300 + 2 * s + c, s, c, bits, c422) for (s, c) in ic.VARIANTS]
    want, want_co = [], []
    for c in pics:
        w, co = [p.copy() for p in c["planes"]], c["coeffs"].copy()
        hh.oracle_intra(checker, bits, c["rec"], co, c["nnzc"], mb_w, mb_h, *w, c422=c422)
        want.append(w)
        want_co.append(co)
    cat = lambda k: np.concatenate([c[k] for c in pics])
    planes = [np.concatenate([c["planes"][i] for c in pics]) for i in range(3)]
    d = [_dev(v) for v in [cat("rec"), cat("coeffs"), cat("nnzc")] + planes]
    fn = gpu.lib.ff_h264_intra_mb_batch_422_cuda if c422 else gpu.lib.ff_h264_intra_mb_batch_hbd_cuda
    gpu.check(fn(bits, d[0].ptr, mb_w, mb_h, len(pics), d[1].ptr, 768, d[2].ptr, d[3].ptr, d[4].ptr, d[5].ptr, planes[0].strides[0],
                 planes[1].strides[0], None))
    device.sync()
    for i, name in enumerate(("y", "cb", "cr")):
        got, w = d[3 + i].download(planes[i].dtype, planes[i].shape), np.concatenate([x[i] for x in want])
        assert np.array_equal(got, w), (name, np.argwhere(got != w)[:5].tolist())
    co = d[1].download(want_co[0].dtype, (len(pics) * mb_w * mb_h, 768))
    assert np.array_equal(co, np.concatenate(want_co)), np.argwhere(co != np.concatenate(want_co))[:5].tolist()


# ---- the flush point ----
def flush_case(mb_w, mb_h, P):
    """P pictures of test_gpu_h264flush.picture_work whose intra macroblocks are the sliced, constrained-intra ones of this file"""
    from test_gpu_h264flush import picture_work
    works = []
    for k in range(P):
        w = picture_work(mb_w, mb_h, 500 + 100 * k, 0.0)
        c = ic.intra_case(mb_w, mb_h, 600 + k, True, True)
        intra = c["rec"]["kind"] != 0
        w["res"]["luma_mode"][intra] = 3
        w["res"]["chroma"][intra] = 0
        w["coeffs"][intra], w["nnzc"][intra], w["intra"] = c["coeffs"][intra], c["nnzc"][intra], c["rec"]
        works.append(w)
    refs = [synth.h264_picture(mb_w, mb_h, seed=11), synth.h264_picture(mb_w, mb_h, seed=12)]
    return works, [synth.h264_picture(mb_w, mb_h, seed=80 + k) for k in range(P)], refs


def test_flush_with_sliced_constrained_intra(gpu, checker):
    from libav_b200 import device
    from test_gpu_h264flush import oracle_chain
    mb_w, mb_h, P = 20, 12, 2
    works, pics, refs = flush_case(mb_w, mb_h, P)
    want, want_co = [], []
    for w, p in zip(works, pics):
        wp = [x.copy() for x in p]
        want_co.append(oracle_chain(checker, w, refs, mb_w, mb_h, *wp))
        want.append(wp)
    work, d, dv = flush_batch(works, pics, refs, mb_w, mb_h)
    gpu.check(gpu.lib.ff_h264_flush_pictures_cuda(C.byref(work), None))
    device.sync()
    d.check([np.concatenate([w[i] for w in want]) for i in range(3)])
    assert np.array_equal(dv["co"].download(np.int16, (mb_w * mb_h * P, 768)), np.concatenate(want_co))


def test_flush_refuses_an_intra_arena_before_its_first_stage(gpu):
    """an arena at +2 bytes, which the residual stage would take: the intra stage cannot, so nothing runs and the planes stay as they were"""
    from libav_b200 import device
    mb_w, mb_h, P = 20, 12, 2
    works, pics, refs = flush_case(mb_w, mb_h, P)
    work, d, dv = flush_batch(works, pics, refs, mb_w, mb_h)
    co = dv["co"].download(np.uint8, (dv["co"].nbytes,))
    work.coeffs = dv["co"].ptr + 2
    refused(gpu, gpu.lib.ff_h264_flush_pictures_cuda(C.byref(work), None), "4-byte aligned")
    device.sync()
    d.check([np.concatenate([p[i] for p in pics]) for i in range(3)], "refused flush")
    assert np.array_equal(dv["co"].download(np.uint8, co.shape), co)
