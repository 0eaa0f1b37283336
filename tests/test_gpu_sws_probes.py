"""The two ceiling probes of the fused same-size yuv420p -> rgb24 call (sws_tma_probe, tools/sws4k_ceiling.py) move exactly the bytes
they stand for: the flat stream reads the batch's Y, U and V planes once and writes every output byte, the move-only kernel stores the
luma rows it staged in the real kernel's tile layout.  Their pictures are wrong on purpose; these tests check the byte flow."""
import numpy as np
import pytest

from libav_b200 import synth

pytestmark = pytest.mark.gpu
FLAGS = 4 | 0x40000 | 0x80000


def _run(gpu, probe, w, h, K):
    from libav_b200 import device
    frames = [synth.yuv420p_frame(w, h, 50 + k) for k in range(K)]
    planes = [np.concatenate([f[p].reshape(-1) for f in frames]) for p in range(3)]
    ysz, csz, osz = w * h, (w // 2) * (h // 2), w * h * 3
    gpu.lib.avb200_set_tuning(b"sws_tma_probe", probe)
    try:
        ctx = device.SwsContext(w, h, w, h, device.PIX_FMT_RGB24, FLAGS)
        d = [device.DevBuf.from_numpy(p) for p in planes]
        d_o = device.DevBuf(osz * K)
        d_o.upload(np.full(osz * K, 0xA5, np.uint8))
        ctx.scale_device([x.ptr for x in d], [w, w // 2, w // 2], [d_o.ptr], [w * 3], nframes=K, src_frame=[ysz, csz, csz], dst_frame=[osz])
        device.sync()
        ctx.close()
    finally:
        gpu.lib.avb200_set_tuning(b"sws_tma_probe", 0)
    return planes, d_o.download(np.uint8, (K, h, w * 3))


def test_flat_stream_probe_reads_every_input_byte_and_writes_every_output_byte(gpu):
    planes, got = _run(gpu, 2, 512, 64, 3)
    src = np.concatenate(planes)                    # 1.5 B/px in, 3 B/px out: the input lands in each half of the output
    assert np.array_equal(got.reshape(-1), np.concatenate([src, src]))


def test_move_probe_stores_the_staged_luma_in_the_tile_layout(gpu):
    w, h, K = 512, 64, 2
    planes, got = _run(gpu, 1, w, h, K)
    y = planes[0].reshape(K, h, w)
    want = np.empty_like(got)
    for f in range(K):
        for r0 in range(0, h, 4):                   # a bulk store = 4 rows x 768 bytes of one 256-pixel tile
            for tx in range(w // 256):
                quarter = y[f, r0:r0 + 4, 256 * tx:256 * tx + 256].reshape(-1)
                want[f, r0:r0 + 4, 768 * tx:768 * tx + 768] = np.tile(quarter, 3).reshape(4, 768)
    assert np.array_equal(got, want)
