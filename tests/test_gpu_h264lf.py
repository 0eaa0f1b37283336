"""GPU parity for the deblocking-decision kernel (SURVEY 8f rank 1): ff_h264_deblock_params_cuda against the CPU
checker (the reference's own h264_loopfilter.c with recording slots when oracle/_ref is present, else the port) on
random decoder side information, record for record; then the whole device chain decisions -> deblocking wavefront
against the oracle's filters driven by the oracle's decisions."""
import ctypes as C

import numpy as np
import pytest

from libav_b200 import synth, tables
from oracle.loader import ptr
import h264_util as hu
from test_oracle_h264lf_cpu import CASES, run as oracle_run

pytestmark = pytest.mark.gpu


def _dev(a):
    from libav_b200 import device
    return device.DevBuf.from_numpy(np.ascontiguousarray(a))


def device_info(infos, field=0, chroma422=None):
    """(FFH264DeblockInfo, the device buffers it points at) for per-picture dicts of equal geometry, stacked row-wise; slice parameters and
    chroma_qp_table are the first picture's"""
    d0 = infos[0]
    cat = lambda k: np.concatenate([d[k] for d in infos], axis=0)
    keep = {k: _dev(cat(k)) for k in ("mb_type", "qscale", "nnz", "cbp", "slice_table", "mv0", "mv1", "ref0", "ref1")}
    keep["sp"] = _dev(d0["slice_params"]); keep["cq"] = _dev(d0["chroma_qp_table"])
    info = tables.FFH264DeblockInfo(d0["mb_w"], d0["mb_h"], len(infos), keep["mb_type"].ptr, keep["qscale"].ptr, keep["nnz"].ptr,
                                    keep["cbp"].ptr, keep["slice_table"].ptr, (C.c_void_p * 2)(keep["mv0"].ptr, keep["mv1"].ptr),
                                    (C.c_void_p * 2)(keep["ref0"].ptr, keep["ref1"].ptr), keep["sp"].ptr, d0["n_slices"], keep["cq"].ptr,
                                    d0["cabac"], d0["t8x8"], field, chroma422)
    return info, keep


def gpu_params(gpu, infos, field=0, chroma422=None, bits=None):
    """infos: list of per-picture dicts of equal geometry (stacked row-wise into one call); bits: through ff_h264_deblock_params_hbd_cuda"""
    from libav_b200 import device
    d0 = infos[0]
    info, keep = device_info(infos, field, chroma422)
    n = d0["mb_w"] * d0["mb_h"] * len(infos)
    out = device.DevBuf(n * 104); out.fill(0xAB)
    if bits is None:
        gpu.check(gpu.lib.ff_h264_deblock_params_cuda(C.byref(info), out.ptr, None))
    else:
        gpu.check(gpu.lib.ff_h264_deblock_params_hbd_cuda(bits, C.byref(info), out.ptr, None))
    device.sync()
    return out.download(np.uint8, (n, 104)), out


def test_field_picture_decisions(gpu, checker):
    """FFH264DeblockInfo.field_picture: the fields of a PAFF frame as pictures of their own (h264_loopfilter.c:551-557,723)"""
    from test_oracle_h264lf_cpu import FIELD_CASES, as_field
    for case in FIELD_CASES:
        for (mw, mh) in ((11, 9), (2, 5), (40, 17)):
            d = as_field(synth.h264_deblock_info(mw, mh, **case))
            try:
                checker.h264_deblock_picture_structure(1)
                want = oracle_run(checker, d)
            finally:
                checker.h264_deblock_picture_structure(0)
            got, _ = gpu_params(gpu, [d], field=1)
            bad = np.argwhere((got[:, :102] != want[:, :102]).any(axis=1))
            assert not len(bad), (case, mw, mh, bad[:4].ravel().tolist(), got[bad[0, 0]].tolist(), want[bad[0, 0]].tolist())


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join("%s%s" % kv for kv in c.items()))
def test_decisions_match_checker(gpu, checker, case):
    for (mw, mh) in ((11, 9), (1, 1), (2, 5), (40, 23)):
        d = synth.h264_deblock_info(mw, mh, **case)
        want = oracle_run(checker, d)
        got, _ = gpu_params(gpu, [d])
        bad = np.argwhere((got[:, :102] != want[:, :102]).any(axis=1))
        assert not len(bad), (mw, mh, bad[:4].ravel().tolist(), got[bad[0, 0]].tolist(), want[bad[0, 0]].tolist())


def test_full_hd_batch_of_pictures(gpu, checker):
    """config-3 geometry, 3 stacked pictures with the same slice parameters: no decision crosses a picture boundary"""
    infos = [synth.h264_deblock_info(120, 68, seed=20 + k, n_slices=8, bipred=bool(k & 1), mode=1) for k in range(3)]
    for d in infos[1:]:
        d["slice_params"] = infos[0]["slice_params"]; d["chroma_qp_table"] = infos[0]["chroma_qp_table"]
    for d in infos:                                  # list_count comes from the shared slice parameters
        d["slice_params"] = infos[0]["slice_params"]
    got, _ = gpu_params(gpu, infos)
    want = np.concatenate([oracle_run(checker, d) for d in infos])
    assert np.array_equal(got[:, :102], want[:, :102])


def test_decisions_feed_the_deblocking_wavefront(gpu, checker):
    """device chain: side information -> records -> filtered picture, with no host round trip in between"""
    from libav_b200 import device
    mw, mh = 20, 12
    d = synth.h264_deblock_info(mw, mh, seed=31, n_slices=4, bipred=True, t8x8=1, cabac=0)
    y, cb, cr = synth.h264_picture(mw, mh, seed=6)
    want_rec = oracle_run(checker, d).view(synth.DEBLOCK_DT).reshape(-1)
    wy, wcb, wcr = y.copy(), cb.copy(), cr.copy()
    hu.oracle_deblock(checker, want_rec, mw, mh, wy, wcb, wcr)
    _, d_rec = gpu_params(gpu, [d])
    dy, dcb, dcr = _dev(y), _dev(cb), _dev(cr)
    prog = device.DevBuf(4 * 2 * mh); prog.fill(0)
    gpu.check(gpu.lib.ff_h264_deblock_picture_cuda(d_rec.ptr, mw, mh, dy.ptr, dcb.ptr, dcr.ptr, y.strides[0], cb.strides[0], prog.ptr, None))
    device.sync()
    assert np.array_equal(dy.download(np.uint8, y.shape), wy)
    assert np.array_equal(dcb.download(np.uint8, cb.shape), wcb)
    assert np.array_equal(dcr.download(np.uint8, cr.shape), wcr)
    assert (wy != y).mean() > 0.001          # noise pictures rarely pass the |p0 - q0| < alpha gate
