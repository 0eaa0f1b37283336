"""GPU parity of the same-size yuv420p -> rgb24 / bgr24 fast path (config 5's kernel): the TMA-staged kernel of csrc/sws_fused_tma.cu
and the LDG kernel that planes a tensor map cannot describe fall back to, byte for byte against the CPU checker (the compiled
reference's sws_scale when oracle/_ref exists): ragged widths (not a multiple of the 256-pixel tile), heights whose row pairs do not
fill the last 8-row tile, the clamped chroma windows at the top and bottom of the plane, multi-frame device batches (every frame
compared), the banded host-pointer call, and back-to-back dependent launches into one output."""
import ctypes as C

import numpy as np
import pytest

from libav_b200 import synth
from oracle.loader import ptr

pytestmark = pytest.mark.gpu
FLAGS = 4 | 0x40000 | 0x80000

# byte offset of the device chroma planes -> which kernel runs: 16-byte aligned planes go through the TMA kernel; chroma planes 8 bytes
# off still pass the LDG kernel's alignment check but not the tensor maps', so sws_fused_rgb24_v3_kernel runs
VARIANTS = {"tma": 0, "ldg": 8}


def oracle_packed(o, yuv, w, h, fmt):
    dst = [np.zeros((h, w * 3), np.uint8)]
    sp = (C.c_void_p * 3)(*[a.ctypes.data for a in yuv]); ss = (C.c_int * 3)(*[a.strides[0] for a in yuv])
    dp = (C.c_void_p * 3)(dst[0].ctypes.data, None, None); ds = (C.c_int * 3)(w * 3, 0, 0)
    assert o.sws_planar(0, sp, ss, w, h, fmt, dp, ds, w, h, FLAGS) == h
    return dst[0]


def upload_frames(frames, chroma_offset=0):
    """device planes of len(frames) frames laid out frame after frame, the chroma planes `chroma_offset` bytes into their buffers:
    (the buffers, which the caller keeps alive, and the three plane pointers)"""
    from libav_b200 import device
    planes = [np.concatenate([f[p].reshape(-1) for f in frames]) for p in range(3)]
    pad = np.zeros(chroma_offset, np.uint8)
    bufs = [device.DevBuf.from_numpy(planes[0])] + [device.DevBuf.from_numpy(np.concatenate([pad, c])) for c in planes[1:]]
    return bufs, [bufs[0].ptr, bufs[1].ptr + chroma_offset, bufs[2].ptr + chroma_offset]


def device_frames(ctx, frames, w, h, chroma_offset=0):
    """the device-pointer batch call over len(frames) frames laid out frame after frame"""
    from libav_b200 import device
    K = len(frames)
    ysz, csz, osz = w * h, (w // 2) * (h // 2), w * h * 3
    bufs, src = upload_frames(frames, chroma_offset)
    d_o = device.DevBuf(osz * K)
    d_o.upload(np.full(osz * K, 0xA5, np.uint8))
    ctx.scale_device(src, [w, w // 2, w // 2], [d_o.ptr], [w * 3], nframes=K, src_frame=[ysz, csz, csz], dst_frame=[osz])
    device.sync()
    return d_o.download(np.uint8, (K, h, w * 3))


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("w,h", [(640, 480), (1936, 1082), (272, 66), (256, 16), (3840, 2160), (4096, 2176), (528, 24)])
def test_fused_variants_match_the_reference(gpu, checker, variant, w, h):
    from libav_b200 import device
    for fmt in (device.PIX_FMT_RGB24, device.PIX_FMT_BGR24):
        yuv = synth.yuv420p_frame(w, h, 3 + w + fmt)
        ctx = device.SwsContext(w, h, w, h, fmt, FLAGS)
        assert ctx.fused
        want = oracle_packed(checker, yuv, w, h, fmt)
        assert np.array_equal(device_frames(ctx, [yuv], w, h, VARIANTS[variant])[0], want), "device call"
        if variant == "tma":            # the host call stages the planes itself
            assert np.array_equal(ctx.scale(yuv), want), "host call (banded above 64 rows)"
        ctx.close()


def test_extreme_samples_and_flat_pictures(gpu, checker):
    """all-0 / all-255 planes and the four corners of (Y, U, V) drive the chroma FIR to its overshoot (the clip in front of the term
    tables) and the output stage to both ends of its clip"""
    from libav_b200 import device
    w, h = 512, 64
    r = np.random.RandomState(5)
    cases = []
    for yv, uv, vv in ((0, 0, 0), (255, 255, 255), (0, 255, 0), (255, 0, 255), (16, 128, 128), (235, 240, 16)):
        cases.append([np.full((h, w), yv, np.uint8), np.full((h // 2, w // 2), uv, np.uint8), np.full((h // 2, w // 2), vv, np.uint8)])
    cases.append([r.choice([0, 255], (h, w)).astype(np.uint8), r.choice([0, 255], (h // 2, w // 2)).astype(np.uint8), r.choice([0, 255], (h // 2, w // 2)).astype(np.uint8)])
    for variant, offset in VARIANTS.items():
        ctx = device.SwsContext(w, h, w, h, device.PIX_FMT_RGB24, FLAGS)
        got = device_frames(ctx, cases, w, h, offset)
        for k, yuv in enumerate(cases):
            assert np.array_equal(got[k], oracle_packed(checker, yuv, w, h, device.PIX_FMT_RGB24)), (variant, k)
        ctx.close()


def test_config5_batch_every_frame_against_the_reference(gpu, checker):
    """config 5's per-GPU batch as bench.py launches it: 16 4K frames in one launch, each of them compared with the checker, in rgb24
    and bgr24"""
    from libav_b200 import device
    w, h, K = 3840, 2160, 16
    frames = [synth.yuv420p_frame(w, h, 1 + k) for k in range(K)]
    for fmt in (device.PIX_FMT_RGB24, device.PIX_FMT_BGR24):
        ctx = device.SwsContext(w, h, w, h, fmt, FLAGS)
        out = device_frames(ctx, frames, w, h)
        ctx.close()
        if fmt == device.PIX_FMT_RGB24:
            assert synth.crc32_ieee_be(out[0].tobytes()) == 0xE1558C0A          # SURVEY 8d's known answer for the seed-1 frame
        for k in range(K):
            assert np.array_equal(out[k], oracle_packed(checker, frames[k], w, h, fmt)), (fmt, k)


@pytest.mark.parametrize("fmt_name", ["rgb24", "bgr24"])
def test_ragged_width_and_last_tile_row(gpu, checker, fmt_name):
    """1000 x 700: a last tile 232 pixels wide and a last tile row of two row pairs, three frames in one call"""
    from libav_b200 import device
    fmt = device.PIX_FMT_RGB24 if fmt_name == "rgb24" else device.PIX_FMT_BGR24
    w, h = 1000, 700
    frames = [synth.yuv420p_frame(w, h, s) for s in (40, 41, 42)]
    ctx = device.SwsContext(w, h, w, h, fmt, FLAGS)
    got = device_frames(ctx, frames, w, h)
    ctx.close()
    for k, f in enumerate(frames):
        assert np.array_equal(got[k], oracle_packed(checker, f, w, h, fmt)), "frame %d" % k


@pytest.mark.parametrize("h", [64, 66, 1080, 1082])
def test_host_call_bands(gpu, checker, h):
    """sws_scale_cuda sends a frame of 64 rows or more through in three row bands of whole tiles on three streams: equal bands (1080),
    a shorter last band (64: 12 / 12 / 8 row pairs, 66: 12 / 12 / 9, 1082: 184 / 184 / 173); two calls on one context"""
    from libav_b200 import device
    w = 1920
    yuv = synth.yuv420p_frame(w, h, 77)
    want = oracle_packed(checker, yuv, w, h, device.PIX_FMT_RGB24)
    ctx = device.SwsContext(w, h, w, h, device.PIX_FMT_RGB24, FLAGS)
    for _ in range(2):
        assert np.array_equal(ctx.scale(yuv, fill=0x5A), want)
    ctx.close()


def test_host_bands_start_mid_picture(gpu, checker):
    """the host-pointer call sends a 4K bgr24 frame through in three row bands: the second and third launches start at row pairs 360
    and 720"""
    from libav_b200 import device
    w, h = 3840, 2160
    yuv = synth.yuv420p_frame(w, h, 7)
    want = oracle_packed(checker, yuv, w, h, device.PIX_FMT_BGR24)
    ctx = device.SwsContext(w, h, w, h, device.PIX_FMT_BGR24, FLAGS)
    got = ctx.scale(yuv, fill=0x5A)
    ctx.close()
    assert np.array_equal(got, want)


def test_back_to_back_launches_into_one_output(gpu, checker):
    """two launches on one stream without a synchronisation between them write the same output batch: the second picture is what
    remains (a dependent launch must not store before the launch ahead of it has finished)"""
    from libav_b200 import device
    w, h, K = 3840, 2160, 4
    ysz, csz, osz = w * h, (w // 2) * (h // 2), w * h * 3
    frames = [synth.yuv420p_frame(w, h, 1 + k) for k in range(2 * K)]
    ctx = device.SwsContext(w, h, w, h, device.PIX_FMT_RGB24, FLAGS)
    sets = [upload_frames(frames[:K]), upload_frames(frames[K:])]
    d_o = device.DevBuf(osz * K)
    for _, src in sets:
        ctx.scale_device(src, [w, w // 2, w // 2], [d_o.ptr], [w * 3], nframes=K, src_frame=[ysz, csz, csz], dst_frame=[osz])
    device.sync()
    got = d_o.download(np.uint8, (K, h, w * 3))
    ctx.close()
    for k in range(K):
        assert np.array_equal(got[k], oracle_packed(checker, frames[K + k], w, h, device.PIX_FMT_RGB24)), "frame %d" % k


def test_colorspace_details_reach_the_term_tables(gpu, checker):
    """sws_setColorspaceDetails changes the constants the CTA builds its tables from"""
    from libav_b200 import device
    w, h = 768, 96
    yuv = synth.yuv420p_frame(w, h, 9)
    for tab, rng, bri, con, sat in (((117504, 138453, 13954, 34903), 1, 0, 1 << 16, 1 << 16),      # ff_yuv2rgb_coeffs[SWS_CS_ITU709], full range
                                    ((117579, 136230, 16907, 35559), 1, -4000, 60000, 80000)):     # SMPTE 240M + brightness / contrast / saturation
        t = (C.c_int * 4)(*tab)
        ctx = device.SwsContext(w, h, w, h, device.PIX_FMT_RGB24, FLAGS)
        assert gpu.lib.sws_setColorspaceDetails_cuda(ctx.ctx, t, rng, t, 0, bri, con, sat) == 0
        checker.sws_set_colorspace(t, rng, bri, con, sat)
        try:
            want = oracle_packed(checker, yuv, w, h, device.PIX_FMT_RGB24)
        finally:
            checker.sws_set_colorspace(None, 0, 0, 0, 0)
        assert np.array_equal(device_frames(ctx, [yuv], w, h)[0], want), tab
        ctx.close()
