"""GPU parity of every shape of the TMA-staged same-size yuv420p -> rgb24 / bgr24 kernel (csrc/sws_fused_tma.cu): 2 or 3 tile stages per
warp, with or without L2 evict-first hints, launched plainly or as a programmatic dependent of the launch before it, 4 / 12 / 14 warps
per CTA, term tables or arithmetic terms -- byte for byte against the CPU checker on config 5's 16-frame 4K batch (with its known
answer), a ragged width, the banded host call whose launches start mid-picture, and back-to-back launches into one output.  The ceiling
probes (sws_tma_probe) write wrong pictures on purpose and are checked in test_gpu_sws_probes.py."""
import ctypes as C
import zlib

import numpy as np
import pytest

from libav_b200 import synth

pytestmark = pytest.mark.gpu
FLAGS = 4 | 0x40000 | 0x80000
KNOBS = ("sws_tma_stages", "sws_tma_hint", "sws_tma_pdl", "sws_tma_warps", "sws_tma_lut", "sws_tma_probe", "sws_fused_variant",
         "sws_host_bands")

SHAPES = {
    "default": {},                                                          # 3 stages, hints, dependent launch
    "before": {"sws_tma_stages": 2, "sws_tma_hint": 1, "sws_tma_pdl": 1},  # the kernel without the three
    "stages2": {"sws_tma_stages": 2},
    "no_hint": {"sws_tma_hint": 1},
    "no_pdl": {"sws_tma_pdl": 1},
    "warps4": {"sws_tma_warps": 4},                                        # 3 stages, two CTAs per SM
    "warps14": {"sws_tma_warps": 14},                                      # 3 stages do not fit: 2
    "arith": {"sws_tma_lut": 2},
}
_REF, _FRAMES = {}, {}


def _set(gpu, knobs):
    for k in KNOBS:
        gpu.lib.avb200_set_tuning(k.encode(), int(knobs.get(k, 0)))


def _oracle(o, yuv, w, h, fmt):
    dst = np.zeros((h, w * 3), np.uint8)
    sp = (C.c_void_p * 3)(*[a.ctypes.data for a in yuv]); ss = (C.c_int * 3)(*[a.strides[0] for a in yuv])
    dp = (C.c_void_p * 3)(dst.ctypes.data, None, None); ds = (C.c_int * 3)(w * 3, 0, 0)
    assert o.sws_planar(0, sp, ss, w, h, fmt, dp, ds, w, h, FLAGS) == h
    return dst


def _frames(w, h, seeds):
    """the synthetic frames of the seeds (made once per geometry: a 4K frame takes about a second)"""
    key = (w, h, tuple(seeds))
    if key not in _FRAMES:
        _FRAMES[key] = [synth.yuv420p_frame(w, h, s) for s in seeds]
    return _FRAMES[key]


def _ref_crcs(checker, w, h, seeds, fmt):
    """CRC-32 of the checker's picture of each seed's frame (computed once per geometry and format)"""
    key = (w, h, tuple(seeds), fmt)
    if key not in _REF:
        _REF[key] = [zlib.crc32(_oracle(checker, f, w, h, fmt).tobytes()) for f in _frames(w, h, seeds)]
    return _REF[key]


def _device_batch(ctx, frames, w, h):
    from libav_b200 import device
    K = len(frames)
    ysz, csz, osz = w * h, (w // 2) * (h // 2), w * h * 3
    d = [device.DevBuf.from_numpy(np.concatenate([f[p].reshape(-1) for f in frames])) for p in range(3)]
    d_o = device.DevBuf(osz * K)
    d_o.upload(np.full(osz * K, 0xA5, np.uint8))
    ctx.scale_device([x.ptr for x in d], [w, w // 2, w // 2], [d_o.ptr], [w * 3], nframes=K, src_frame=[ysz, csz, csz], dst_frame=[osz])
    device.sync()
    return d_o.download(np.uint8, (K, h, w * 3))


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("fmt_name", ["rgb24", "bgr24"])
def test_config5_batch(gpu, checker, shape, fmt_name):
    """config 5's launch: 16 distinct 4K frames in one device-pointer call, every frame against the checker; frame 0 (seed 1) of the
    rgb24 batch is SURVEY 8d's known answer"""
    from libav_b200 import device
    fmt = device.PIX_FMT_RGB24 if fmt_name == "rgb24" else device.PIX_FMT_BGR24
    w, h, seeds = 3840, 2160, list(range(1, 17))
    want = _ref_crcs(checker, w, h, seeds, fmt)
    _set(gpu, SHAPES[shape])
    try:
        ctx = device.SwsContext(w, h, w, h, fmt, FLAGS)
        assert ctx.fused
        got = _device_batch(ctx, _frames(w, h, seeds), w, h)
        ctx.close()
    finally:
        _set(gpu, {})
    if fmt == device.PIX_FMT_RGB24:
        assert synth.crc32_ieee_be(got[0].tobytes()) == 0xE1558C0A
    for k in range(len(seeds)):
        assert zlib.crc32(got[k].tobytes()) == want[k], "frame %d" % k


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("fmt_name", ["rgb24", "bgr24"])
def test_ragged_width_and_last_tile_row(gpu, checker, shape, fmt_name):
    """1000 x 700: a last tile 232 pixels wide and a last tile row of two row pairs, three frames in one call"""
    from libav_b200 import device
    fmt = device.PIX_FMT_RGB24 if fmt_name == "rgb24" else device.PIX_FMT_BGR24
    w, h = 1000, 700
    frames = _frames(w, h, [40, 41, 42])
    _set(gpu, SHAPES[shape])
    try:
        ctx = device.SwsContext(w, h, w, h, fmt, FLAGS)
        got = _device_batch(ctx, frames, w, h)
        ctx.close()
    finally:
        _set(gpu, {})
    for k, f in enumerate(frames):
        assert np.array_equal(got[k], _oracle(checker, f, w, h, fmt)), "frame %d" % k


@pytest.mark.parametrize("shape", list(SHAPES))
def test_host_bands_start_mid_picture(gpu, checker, shape):
    """the host-pointer call sends a 4K frame through in three row bands: the second and third launches start at row pairs 360 and 720"""
    from libav_b200 import device
    w, h = 3840, 2160
    yuv = _frames(w, h, [7])[0]
    want = _oracle(checker, yuv, w, h, device.PIX_FMT_BGR24)
    _set(gpu, dict(SHAPES[shape], sws_host_bands=3))
    try:
        ctx = device.SwsContext(w, h, w, h, device.PIX_FMT_BGR24, FLAGS)
        got = ctx.scale(yuv, fill=0x5A)
        ctx.close()
    finally:
        _set(gpu, {})
    assert np.array_equal(got, want)


@pytest.mark.parametrize("shape", ["default", "before"])
def test_back_to_back_launches_into_one_output(gpu, checker, shape):
    """two launches on one stream without a synchronisation between them write the same output batch: the second picture is what
    remains (a dependent launch must not store before the launch ahead of it has finished)"""
    from libav_b200 import device
    w, h, K = 3840, 2160, 4
    ysz, csz, osz = w * h, (w // 2) * (h // 2), w * h * 3
    sets = [_frames(w, h, list(range(1, 17)))[:K], _frames(w, h, list(range(1, 17)))[K:2 * K]]
    want = _ref_crcs(checker, w, h, list(range(1, 17)), device.PIX_FMT_RGB24)[K:2 * K]
    _set(gpu, SHAPES[shape])
    try:
        ctx = device.SwsContext(w, h, w, h, device.PIX_FMT_RGB24, FLAGS)
        srcs = [[device.DevBuf.from_numpy(np.concatenate([f[p].reshape(-1) for f in fr])) for p in range(3)] for fr in sets]
        d_o = device.DevBuf(osz * K)
        for d in srcs:
            ctx.scale_device([x.ptr for x in d], [w, w // 2, w // 2], [d_o.ptr], [w * 3], nframes=K, src_frame=[ysz, csz, csz], dst_frame=[osz])
        device.sync()
        got = d_o.download(np.uint8, (K, h, w * 3))
        ctx.close()
    finally:
        _set(gpu, {})
    for k in range(K):
        assert zlib.crc32(got[k].tobytes()) == want[k], "frame %d" % k
