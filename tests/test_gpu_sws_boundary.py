"""Consecutive launches of the TMA-staged fused yuv420p -> rgb24 / bgr24 kernel (csrc/sws_fused_tma.cu): each launch is a dependent of
the one ahead of it on the stream, and hands out its tiles past the first eight per warp from a tile counter that it leaves at zero for
the next launch on that stream.  Every frame is compared with the CPU checker."""
import ctypes as C

import numpy as np
import pytest

from libav_b200 import synth

pytestmark = pytest.mark.gpu
FLAGS = 4 | 0x40000 | 0x80000


def want_of(o, yuv, w, h, fmt):
    dst = np.zeros((h, w * 3), np.uint8)
    sp = (C.c_void_p * 3)(*[a.ctypes.data for a in yuv]); ss = (C.c_int * 3)(*[a.strides[0] for a in yuv])
    dp = (C.c_void_p * 3)(dst.ctypes.data, None, None); ds = (C.c_int * 3)(w * 3, 0, 0)
    assert o.sws_planar(0, sp, ss, w, h, fmt, dp, ds, w, h, FLAGS) == h
    return dst


def planes_of(torch, frames):
    return [torch.from_numpy(np.concatenate([f[p].reshape(-1) for f in frames])).cuda() for p in range(3)]


def launch(ctx, src, out, w, h, K, stream):
    ysz, csz = w * h, (w // 2) * (h // 2)
    ctx.scale_device([p.data_ptr() for p in src], [w, w // 2, w // 2], [out.data_ptr()], [w * 3], nframes=K,
                     src_frame=[ysz, csz, csz], dst_frame=[w * h * 3], stream=stream)


@pytest.mark.parametrize("fmt_name", ["rgb24", "bgr24"])
def test_input_rewritten_just_before_the_launch(gpu, checker, fmt_name):
    """A copy kernel on the same stream overwrites the Y / U / V planes right before each launch, while the launch ahead of it may
    still run: a launch that read the planes before the copy had finished would write the old pictures."""
    import torch
    from libav_b200 import device
    fmt = device.PIX_FMT_RGB24 if fmt_name == "rgb24" else device.PIX_FMT_BGR24
    w, h, K = 3840, 2160, 4
    sets = [[synth.yuv420p_frame(w, h, 100 + 8 * s + k) for k in range(K)] for s in range(3)]
    staged = [planes_of(torch, fr) for fr in sets]
    src = [torch.empty_like(p) for p in staged[0]]
    outs = [torch.empty(w * h * 3 * K, dtype=torch.uint8, device="cuda") for _ in range(3)]
    ctx = device.SwsContext(w, h, w, h, fmt, FLAGS)
    stream = torch.cuda.current_stream()
    torch.cuda.synchronize()
    for s in range(3):
        for dst, p in zip(src, staged[s]):
            dst.copy_(p)
        launch(ctx, src, outs[s], w, h, K, stream.cuda_stream)
    torch.cuda.synchronize()
    ctx.close()
    for s in range(3):
        got = outs[s].view(K, h, w * 3).cpu().numpy()
        for k in range(K):
            assert np.array_equal(got[k], want_of(checker, sets[s][k], w, h, fmt)), (s, k)


def test_mixed_batch_sizes_on_one_context(gpu, checker):
    """Seven launches back to back on one context with 1, 16, 3, 1, 16, 3, 1 frames: 4K launches of 1 and 3 frames take the
    4-warp CTAs (fewer than 24 tiles per SM), 16 frames the 12-warp CTAs; 1 frame has too few tiles for the counter, 3 and 16 frames
    take tiles from it, and each launch must leave it at zero for the next."""
    import torch
    from libav_b200 import device
    w, h = 3840, 2160
    frames = [synth.yuv420p_frame(w, h, 200 + k) for k in range(2)]
    wants = [want_of(checker, f, w, h, device.PIX_FMT_RGB24) for f in frames]
    src = planes_of(torch, [frames[k % 2] for k in range(16)])
    ks = [1, 16, 3, 1, 16, 3, 1]
    outs = [torch.full((w * h * 3 * K,), 0x5A, dtype=torch.uint8, device="cuda") for K in ks]
    ctx = device.SwsContext(w, h, w, h, device.PIX_FMT_RGB24, FLAGS)
    stream = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    for K, out in zip(ks, outs):
        launch(ctx, src, out, w, h, K, stream)
    torch.cuda.synchronize()
    for i, (K, out) in enumerate(zip(ks, outs)):
        got = out.view(K, h, w * 3).cpu().numpy()
        for k in range(K):
            assert np.array_equal(got[k], wants[k % 2]), (i, K, k)
    # a second round on the same context: the counter came back to zero after each launch
    for out in outs[:2]:
        out.fill_(0x5A)
    for K, out in zip(ks[:2], outs[:2]):
        launch(ctx, src, out, w, h, K, stream)
    torch.cuda.synchronize()
    ctx.close()
    for K, out in zip(ks[:2], outs[:2]):
        got = out.view(K, h, w * 3).cpu().numpy()
        for k in range(K):
            assert np.array_equal(got[k], wants[k % 2]), ("second round", K, k)


def test_banded_host_call_after_batches(gpu, checker):
    """The host-pointer call sends a 4K picture through in three row bands on the context's own three streams, each band a launch with
    the counter of its stream; here on a context whose caller-stream counter has already served batch launches."""
    import torch
    from libav_b200 import device
    w, h, K = 3840, 2160, 16
    frames = [synth.yuv420p_frame(w, h, 300 + k) for k in range(2)]
    src = planes_of(torch, [frames[k % 2] for k in range(K)])
    out = torch.empty(w * h * 3 * K, dtype=torch.uint8, device="cuda")
    ctx = device.SwsContext(w, h, w, h, device.PIX_FMT_RGB24, FLAGS)
    wants = [want_of(checker, f, w, h, device.PIX_FMT_RGB24) for f in frames]
    for _ in range(2):
        launch(ctx, src, out, w, h, K, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for r in range(3):
        assert np.array_equal(ctx.scale(frames[r % 2], fill=0x5A), wants[r % 2]), r
    out.fill_(0)
    launch(ctx, src, out, w, h, K, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ctx.close()
    got = out.view(K, h, w * 3).cpu().numpy()
    for k in range(K):
        assert np.array_equal(got[k], wants[k % 2]), k
