"""GPU: the deblocking decisions of 9 / 10-bit pictures.  ff_h264_deblock_params_hbd_cuda on side information in the decoder's QP' scale
(synth.h264_deblock_info with bit_depth: qscale 0..51 + qp_bd_offset, I_PCM macroblocks at 0, qp_thresh with its bit-depth term, offsets out
to +-12) against the CPU checker deciding at the same depth (the reference's own h264_loopfilter.c with sps->bit_depth_luma set when
oracle/_ref is present, else the port), record for record; its refusals and its 8-bit identity with ff_h264_deblock_params_cuda; the 9 /
10-bit flush with deblock_info for 4:2:0 (test_zz_gpu_h264_hbd.py) and 4:2:2 pictures; the reference's loop-filter driver over the
product's 9 / 10-bit H264DSPContext slots."""
import ctypes as C

import numpy as np
import pytest

from libav_b200 import synth
from test_gpu_h264lf import device_info, gpu_params
from test_oracle_h264lf_cpu import C422_CASES, CASES, FIELD_CASES, as_field
from test_oracle_h264lf_hbd_cpu import hbd_oracle, run, run422

pytestmark = pytest.mark.gpu
GEOMS = ((1, 1), (2, 5), (11, 9), (40, 23))
ids = lambda c: "-".join("%s%s" % kv for kv in c.items())


@pytest.fixture
def decider(checker):
    """the strongest checker that decides at 9 / 10 bit"""
    return hbd_oracle(checker)


def _same(got, want, what):
    bad = np.argwhere((got != want).any(axis=1))
    assert not len(bad), (what, bad[:4].ravel().tolist(), got[bad[0, 0]].tolist(), want[bad[0, 0]].tolist())


@pytest.mark.parametrize("case", CASES, ids=ids)
@pytest.mark.parametrize("bits", [9, 10])
def test_decisions_hbd(gpu, decider, bits, case):
    for (mw, mh) in GEOMS:
        d = synth.h264_deblock_info(mw, mh, bit_depth=bits, **case)
        got, _ = gpu_params(gpu, [d], bits=bits)
        _same(got, run(decider, d), (mw, mh))


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n_slices", [1, 2, 32])
@pytest.mark.parametrize("bits", [9, 10])
def test_decisions_hbd_slices(gpu, decider, bits, n_slices, mode):
    """1..32 slice numbers (the reference keeps 32 ref2frm tables) under every deblocking_filter mode, P and B"""
    for k, (mw, mh) in enumerate(GEOMS):
        d = synth.h264_deblock_info(mw, mh, seed=40 + k, n_slices=n_slices, mode=mode, bipred=bool(k & 1), t8x8=1, cabac=k & 1, bit_depth=bits)
        got, _ = gpu_params(gpu, [d], bits=bits)
        want = run(decider, d)
        _same(got, want, (mw, mh))
        assert mode or not want.any()


@pytest.mark.parametrize("case", FIELD_CASES, ids=ids)
@pytest.mark.parametrize("bits", [9, 10])
def test_field_picture_decisions_hbd(gpu, decider, bits, case):
    for (mw, mh) in GEOMS:
        d = as_field(synth.h264_deblock_info(mw, mh, bit_depth=bits, **case))
        try:
            decider.h264_deblock_picture_structure(1)
            want = run(decider, d)
        finally:
            decider.h264_deblock_picture_structure(0)
        got, _ = gpu_params(gpu, [d], field=1, bits=bits)
        _same(got, want, (mw, mh))


@pytest.mark.parametrize("case", C422_CASES, ids=ids)
@pytest.mark.parametrize("bits", [9, 10])
def test_chroma422_decisions_hbd(gpu, decider, bits, case):
    """4:2:2: the 104-byte records and the 52-byte records of the four horizontal chroma edges"""
    from libav_b200 import device
    for (mw, mh) in GEOMS:
        d = synth.h264_deblock_info(mw, mh, bit_depth=bits, **case)
        want, want_ext = run422(decider, d)
        ext = device.DevBuf(52 * mw * mh); ext.fill(0xCD)
        got, _ = gpu_params(gpu, [d], chroma422=ext.ptr, bits=bits)
        _same(got, want, (mw, mh))
        _same(ext.download(np.uint8, (mw * mh, 52)), want_ext, ("ext", mw, mh))


@pytest.mark.parametrize("bits", [9, 10])
def test_stacked_pictures_hbd(gpu, decider, bits):
    """three stacked 120x68 pictures with one set of slice headers: no decision crosses a picture boundary"""
    infos = [synth.h264_deblock_info(120, 68, seed=20 + k, n_slices=8, bipred=bool(k & 1), mode=1, bit_depth=bits) for k in range(3)]
    for d in infos[1:]:
        d["slice_params"], d["chroma_qp_table"] = infos[0]["slice_params"], infos[0]["chroma_qp_table"]
    got, _ = gpu_params(gpu, infos, bits=bits)
    _same(got, np.concatenate([run(decider, d) for d in infos]), "stacked")


def test_refusals_leave_the_records_untouched(gpu):
    from libav_b200 import device
    d = synth.h264_deblock_info(11, 9, seed=3, bit_depth=10)
    info, keep = device_info([d])
    out = device.DevBuf(99 * 104); out.fill(0xAB)
    for bits in (0, 7, 11, 12, 16, -1):
        assert gpu.lib.ff_h264_deblock_params_hbd_cuda(bits, C.byref(info), out.ptr, None) == -1, bits
        assert "bit_depth" in gpu.last_error()
        gpu.lib.avb200_clear_error()
    assert gpu.lib.ff_h264_deblock_params_hbd_cuda(10, None, out.ptr, None) == -1
    assert gpu.lib.ff_h264_deblock_params_hbd_cuda(10, C.byref(info), None, None) == -1
    gpu.lib.avb200_clear_error()
    device.sync()
    assert (out.download(np.uint8, (99, 104)) == 0xAB).all()


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_8_bit_equals_the_8_bit_call(gpu, case):
    """bit_depth 8 through the new call: byte for byte what ff_h264_deblock_params_cuda writes, and nothing past the last record"""
    from libav_b200 import device
    for (mw, mh) in GEOMS:
        d = synth.h264_deblock_info(mw, mh, **case)
        n = mw * mh
        info, keep = device_info([d])
        a, b = device.DevBuf((n + 1) * 104), device.DevBuf((n + 1) * 104)
        a.fill(0xAB); b.fill(0xAB)
        gpu.check(gpu.lib.ff_h264_deblock_params_cuda(C.byref(info), a.ptr, None))
        gpu.check(gpu.lib.ff_h264_deblock_params_hbd_cuda(8, C.byref(info), b.ptr, None))
        device.sync()
        ga, gb = a.download(np.uint8, (n + 1, 104)), b.download(np.uint8, (n + 1, 104))
        assert np.array_equal(ga, gb) and (gb[n] == 0xAB).all(), (mw, mh)


@pytest.mark.parametrize("bits", [9, 10])
@pytest.mark.parametrize("mb_w,mb_h,P,p_intra", [(7, 5, 1, 0.0), (20, 12, 2, 0.3)])
def test_flush_422_with_deblock_info(gpu, checker, mb_w, mb_h, P, p_intra, bits):
    """ff_h264_flush_pictures_cuda, chroma_format_idc 2 at 9 / 10 bit, decisions derived from deblock_info: MC -> weighted prediction -> DC
    transforms -> residual -> intra -> decisions (both record arrays compared) -> 4:2:2 loop filter, against the checker chained in that order"""
    from test_zz_gpu_h264_hbd import flush_422
    flush_422(gpu, checker, mb_w, mb_h, P, p_intra, bits, decide=True)


@pytest.mark.parametrize("bits", [9, 10])
def test_loop_filter_slots_under_the_reference_driver_hbd(gpu, refo, bits):
    """the reference's own deblocking driver (h264_loopfilter.c, unmodified, in oracle/_ref) deciding at 9 / 10 bit and filtering uint16
    pictures through the product's 9 / 10-bit H264DSPContext slots: tests/h264_dropin_cases.py"""
    import h264_dropin_cases as D
    if not refo.has("h264_deblock_picture_with_hbd"):
        pytest.skip("oracle/_ref was built before h264_deblock_picture_with_hbd existed")
    assert D.check(refo, gpu.lib, sizes=((6, 4), (1, 1)), bits=bits) == 12
    assert gpu.last_error() == ""
