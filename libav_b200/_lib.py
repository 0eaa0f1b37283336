"""ctypes binding of libavdsp_b200.so (the C-ABI in include/avdsp_b200.h).

Loading fails loudly when the shared library has not been built: there is no Python / CPU fallback for
any op.  Importing this module does not need a GPU (the CPU test suite checks the exported symbols);
calling a compute entry point without an H100 returns -1 and raises AVB200Error.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libavdsp_b200.so")


class AVB200Error(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise AVB200Error("%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(nvcc, sm_90a). There is no fallback path." % LIB_PATH)
    return C.CDLL(LIB_PATH)


lib = _load()

vp, sz, i32, i64 = C.c_void_p, C.c_size_t, C.c_int, C.c_int64
pd = C.c_ssize_t  # ptrdiff_t

# name -> (restype, argtypes); mirrors include/avdsp_b200.h one to one (tests/test_abi_cpu.py parses the
# header and checks that every declared symbol is exported and listed here)
PROTOTYPES = {
    "avb200_device_count": (i32, []),
    "avb200_init": (i32, [i32]),
    "avb200_last_error": (C.c_char_p, []),
    "avb200_clear_error": (None, []),
    "avb200_set_log_callback": (None, [vp]),
    "avb200_set_tuning": (None, [C.c_char_p, i32]),
    "avb200_malloc": (vp, [sz]),
    "avb200_free": (None, [vp]),
    "avb200_host_alloc": (vp, [sz]),
    "avb200_host_free": (None, [vp]),
    "avb200_host_register": (i32, [vp, sz]),
    "avb200_host_unregister": (i32, [vp]),
    "avb200_memcpy_h2d": (i32, [vp, vp, sz, vp]),
    "avb200_memcpy_d2h": (i32, [vp, vp, sz, vp]),
    "avb200_memcpy2d_h2d": (i32, [vp, sz, vp, sz, sz, sz, vp]),
    "avb200_memcpy2d_d2h": (i32, [vp, sz, vp, sz, sz, sz, vp]),
    "avb200_memset": (i32, [vp, i32, sz, vp]),
    "avb200_stream_create": (vp, []),
    "avb200_stream_destroy": (None, [vp]),
    "avb200_stream_sync": (i32, [vp]),
    "avb200_device_sync": (i32, []),
    "avb200_event_create": (vp, []),
    "avb200_event_destroy": (None, [vp]),
    "avb200_event_record": (i32, [vp, vp]),
    "avb200_event_sync": (i32, [vp]),
    "avb200_event_elapsed_ms": (C.c_float, [vp, vp]),
    "ff_simple_idct_batch_cuda": (i32, [i32, vp, vp, vp, pd, sz, i32, i32, vp]),
    "ff_simple_idct10_batch_cuda": (i32, [i32, vp, vp, vp, pd, sz, vp]),
    "ff_xvid_idct_batch_cuda": (i32, [i32, vp, vp, vp, pd, sz, i32, i32, vp]),
    "ff_faanidct_batch_cuda": (i32, [i32, vp, vp, vp, pd, sz, i32, i32, vp]),
    "ff_pixels_clamped_batch_cuda": (i32, [i32, vp, vp, vp, pd, sz, i32, vp]),
    "ff_clear_blocks_batch_cuda": (i32, [vp, sz, vp]),
    "ff_fill_blocks_batch_cuda": (i32, [vp, vp, vp, pd, i32, i32, sz, vp]),
    "ff_simple_idct_batch_host_cuda": (i32, [i32, vp, vp, sz, vp, pd, sz, i32]),
    "ff_h264_idct_add_mb_batch_cuda": (i32, [vp, sz, vp, sz, vp, vp, vp, vp, i32, i32, vp]),
    "ff_h264_mc_batch_cuda": (i32, [vp, sz, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "ff_h264_weight_batch_cuda": (i32, [vp, sz, vp, vp, i32, vp]),
    "ff_h264_deblock_picture_cuda": (i32, [vp, i32, i32, vp, vp, vp, i32, i32, vp, vp]),
    "ff_h264_deblock_batch_cuda": (i32, [vp, i32, i32, i32, vp, vp, vp, i32, i32, vp, vp]),
    "ff_h264_deblock_params_cuda": (i32, [vp, vp, vp]),
    "ff_h264_deblock_params_hbd_cuda": (i32, [i32, vp, vp, vp]),
    "ff_h264_flush_pictures_cuda": (i32, [vp, vp]),
    "ff_h264_dc_dequant_batch_cuda": (i32, [vp, sz, vp, sz, vp, vp]),
    "ff_h264_dc_dequant_batch_422_cuda": (i32, [vp, sz, vp, sz, vp, vp]),
    "ff_h264_intra_mb_batch_cuda": (i32, [vp, i32, i32, i32, vp, sz, vp, vp, vp, vp, i32, i32, vp, vp]),
    "ff_mpeg4_qpel_batch_cuda": (i32, [vp, sz, vp, vp, pd, vp]),
    "ff_pixblock_fdct_batch_cuda": (i32, [i32, vp, vp, vp, vp, pd, vp, sz, vp]),
    "ff_mpeg_dequant_batch_cuda": (i32, [i32, vp, vp, vp, sz, vp]),
    "ff_mpeg_dequant_idct_batch_cuda": (i32, [i32, vp, vp, vp, vp, vp, pd, sz, i32, i32, vp]),
    "ff_mpeg_dequant_xvid_idct_batch_cuda": (i32, [i32, vp, vp, vp, vp, vp, pd, sz, i32, i32, vp]),
    "ff_mpeg_dequant_faanidct_batch_cuda": (i32, [i32, vp, vp, vp, vp, vp, pd, sz, i32, i32, vp]),
    "ff_me_cmp_batch_cuda": (i32, [i32, i32, i32, vp, vp, pd, i32, vp, sz, vp, vp]),
    "ff_h264_idct_add_mb_batch_hbd_cuda": (i32, [i32, i32, vp, sz, vp, sz, vp, vp, vp, vp, i32, i32, vp]),
    "ff_h264_mc_batch_hbd_cuda": (i32, [i32, i32, vp, sz, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "ff_h264_deblock_batch_hbd_cuda": (i32, [i32, vp, i32, i32, i32, vp, vp, vp, i32, i32, vp]),
    "ff_h264_intra_mb_batch_hbd_cuda": (i32, [i32, vp, i32, i32, i32, vp, sz, vp, vp, vp, vp, i32, i32, vp]),
    "ff_h264_intra_mb_batch_422_cuda": (i32, [i32, vp, i32, i32, i32, vp, sz, vp, vp, vp, vp, i32, i32, vp]),
    "ff_h264_weight_batch_hbd_cuda": (i32, [i32, vp, sz, vp, vp, i32, vp]),
    "ff_h264_dc_dequant_batch_hbd_cuda": (i32, [i32, vp, sz, vp, sz, vp, vp]),
    "ff_h264_deblock_batch_422_cuda": (i32, [i32, vp, vp, i32, i32, i32, vp, vp, vp, i32, i32, vp]),
    "ff_me_cmp_enc_state_cuda": (vp, [vp, vp]),
    "ff_me_cmp_enc_state_free_cuda": (None, [vp]),
    "ff_me_cmp_enc_batch_cuda": (i32, [i32, i32, vp, vp, vp, pd, i32, vp, sz, vp, vp, vp]),
    "ff_mpv_quant_state_cuda": (vp, [vp, vp]),
    "ff_mpv_quant_state_free_cuda": (None, [vp]),
    "ff_mpv_dct_quantize_batch_cuda": (i32, [vp, i32, vp, vp, vp, vp, vp, pd, vp, sz, vp, vp, vp, vp]),
    "ff_full_search_cuda": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, vp, vp]),
    "ff_hpel_batch_cuda": (i32, [vp, sz, vp, vp, pd, vp]),
    "ff_mpv_motion_batch_cuda": (i32, [vp, i32, vp, vp]),
    "ff_mpv_flush_pictures_cuda": (i32, [vp, vp]),
    "ff_h263_loop_filter_batch_cuda": (i32, [vp, i32, vp]),
    "ff_fdct_batch_cuda": (i32, [i32, vp, sz, vp]),
    "ff_fft_batch_cuda": (i32, [i32, i32, vp, sz, vp]),
    "ff_mdct_batch_cuda": (i32, [i32, i32, C.c_double, vp, vp, sz, vp]),
    "sws_getContext_cuda": (vp, [i32, i32, i32, i32, i32, i32, i32, vp, vp, vp]),
    "sws_freeContext_cuda": (None, [vp]),
    "sws_setColorspaceDetails_cuda": (i32, [vp, vp, i32, vp, i32, i32, i32, i32]),
    "sws_scale_cuda": (i32, [vp, vp, vp, i32, i32, vp, vp]),
    "sws_scale_frames_cuda": (i32, [vp, vp, vp, vp, vp, vp, vp, i32, vp]),
    "sws_is_fused_cuda": (i32, [vp]),
    "sws_debug_filter_cuda": (i32, [i32, i32, i32, i32, i32, i32, i32, vp, vp, i32, vp]),
    "sws_debug_filter2_cuda": (i32, [i32, i32, i32, i32, i32, i32, i32, vp, vp, vp, vp, i32, vp]),
    "sws_debug_rgb_constants_cuda": (None, [vp]),
    "sws_debug_plan_cuda": (i32, [i32, i32, i32, i32, i32, i32, i32, vp]),
    "sws_debug_slot_view_cuda": (i32, [i32, i32, i32, i32, i32, i32, i32, vp]),
    "ff_idctdsp_init_cuda": (None, [vp, i32, i32, C.c_uint]),
    "ff_xvid_idct_init_cuda": (None, [vp, i32, i32]),
    "ff_blockdsp_init_cuda": (None, [vp]),
    "ff_fdctdsp_init_cuda": (None, [vp, i32, i32, C.c_uint]),
    "ff_me_cmp_init_cuda": (None, [vp]),
    "ff_me_cmp_enc_init_cuda": (i32, [vp, vp, vp]),
    "ff_me_cmp_enc_uninit_cuda": (None, [vp]),
    "ff_mpv_quantize_init_cuda": (i32, [vp, vp, i32]),
    "ff_mpv_quantize_uninit_cuda": (None, [vp]),
    "ff_h264dsp_init_cuda": (None, [vp, i32, i32]),
    "ff_h264qpel_init_cuda": (None, [vp, i32]),
    "ff_h264chroma_init_cuda": (None, [vp, i32]),
    "ff_hpeldsp_init_cuda": (None, [vp, i32]),
    "ff_h264_pred_init_cuda": (None, [vp, i32, i32, i32]),
    "ff_qpeldsp_init_cuda": (None, [vp]),
    "ff_h263dsp_init_cuda": (None, [vp]),
    "ff_mpegvideodsp_init_cuda": (None, [vp]),
    "ff_pixblockdsp_init_cuda": (None, [vp, C.c_uint]),
    "ff_fft_init_cuda": (None, [vp]),
    "ff_mdct_init_cuda": (None, [vp]),
    "ff_sws_init_swscale_cuda": (i32, [vp, vp, vp]),
}

for _name, (_res, _args) in PROTOTYPES.items():
    _f = getattr(lib, _name)
    _f.restype = _res
    _f.argtypes = _args


def last_error():
    return lib.avb200_last_error().decode()


def check(rc, what=""):
    """Raise on a failed call or on a pending sticky error."""
    if rc != 0:
        msg = last_error()
        lib.avb200_clear_error()
        raise AVB200Error("%s failed: %s" % (what or "libavdsp_b200 call", msg or "unknown error"))
    return rc


_initialised = {}


def init(device=0):
    if device not in _initialised:
        check(lib.avb200_init(device), "avb200_init(%d)" % device)
        _initialised[device] = True
        for kv in filter(None, os.environ.get("AVB200_TUNE", "").split(",")):     # test knobs, e.g. mc_variant=2
            k, v = kv.split("=")
            lib.avb200_set_tuning(k.encode(), int(v))
    return True
