"""ctypes loaders for the two CPU oracles.  TEST INFRASTRUCTURE: import only from tests/,
__graft_entry__.smoke() and bench.py's CPU legs.

  port()  oracle/liboracle_port.so   orc_*  plain-C restatement (always buildable with gcc)
  ref()   oracle/_ref/libavref.so    ref_*  the unmodified reference (built where /root/reference exists;
                                            the prebuilt .so travels to the GPU box)
Both expose the prototypes of oracle/oracle_api.h through the same attribute names without prefix.
ref_lib(name) loads one satellite library of the reference, oracle/_ref/lib<name>ref.so; its callers set the prototypes they use.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
PORT_PATH = os.path.join(_HERE, "liboracle_port.so")
REF_PATH = os.path.join(_HERE, "_ref", "libavref.so")
REF_SIMD_PATH = os.path.join(_HERE, "_ref", "libavref_simd.so")

vp, sz, i32, pd, dbl = C.c_void_p, C.c_size_t, C.c_int, C.c_ssize_t, C.c_double

class OrcEncState(C.Structure):
    """oracle_api.h OrcEncState: the MpegEncContext fields quant_psnr / bit / rd read (me_cmp.c:621-782)."""
    _fields_ = [("fdct_sel", C.c_int32), ("dequant", C.c_int32), ("qscale", C.c_int32), ("mb_intra", C.c_int32), ("y_dc_scale", C.c_int32),
                ("c_dc_scale", C.c_int32), ("h263_aic", C.c_int32), ("ac_pred", C.c_int32), ("alternate_scan", C.c_int32),
                ("intra_quant_bias", C.c_int32), ("inter_quant_bias", C.c_int32), ("ac_esc_length", C.c_int32),
                ("intra_matrix", C.c_uint16 * 64), ("inter_matrix", C.c_uint16 * 64),
                ("intra_ac_vlc_length", C.c_void_p), ("intra_ac_vlc_last_length", C.c_void_p), ("inter_ac_vlc_length", C.c_void_p),
                ("inter_ac_vlc_last_length", C.c_void_p), ("luma_dc_vlc_length", C.c_void_p)]


API = {
    "simple_idct_put": (None, [vp, pd, vp]),
    "simple_idct_add": (None, [vp, pd, vp]),
    "simple_idct": (None, [vp]),
    "simple_idct10": (None, [i32, vp, pd, vp]),
    "put_pixels_clamped": (None, [vp, vp, pd]),
    "put_signed_pixels_clamped": (None, [vp, vp, pd]),
    "add_pixels_clamped": (None, [vp, vp, pd]),
    "clear_block": (None, [vp]),
    "clear_blocks": (None, [vp]),
    "fill_block": (None, [i32, vp, C.c_uint8, pd, i32]),
    "idct_batch": (None, [i32, vp, vp, vp, pd, sz, i32]),
    "fdct": (None, [i32, vp]),
    "h264_idct": (None, [i32, vp, vp, i32]),
    "h264_idct_mb": (None, [i32, vp, vp, vp, vp, i32, vp]),
    "h264_luma_dc_dequant_idct": (None, [vp, vp, i32]),
    "h264_chroma_dc_dequant_idct": (None, [vp, i32]),
    "h264_chroma422_dc_dequant_idct": (None, [vp, i32]),
    "h264_loop_filter": (None, [i32, vp, i32, i32, i32, vp]),
    "h264_hbd_idct": (None, [i32, i32, vp, vp, i32]),
    "h264_hbd_idct_mb": (None, [i32, i32, vp, vp, vp, vp, i32, vp]),
    "h264_hbd_dc_dequant": (None, [i32, i32, vp, vp, i32]),
    "h264_hbd_add_pixels_clear": (None, [i32, i32, vp, vp, i32]),
    "h264_hbd_weight": (None, [i32, i32, vp, i32, i32, i32, i32, i32]),
    "h264_hbd_biweight": (None, [i32, i32, vp, vp, i32, i32, i32, i32, i32, i32]),
    "h264_hbd_loop_filter": (None, [i32, i32, vp, i32, i32, i32, vp]),
    "h264_hbd_qpel": (None, [i32, i32, i32, i32, vp, vp, pd]),
    "h264_hbd_chroma": (None, [i32, i32, i32, vp, vp, pd, i32, i32, i32]),
    "h264_hbd_pred": (None, [i32, i32, i32, vp, vp, i32, i32, pd]),
    "h264_hbd_pred_add": (None, [i32, i32, i32, vp, vp, vp, i32, i32, pd]),
    "h264_pred422": (None, [i32, i32, vp, pd]),
    "h264_pred422_add": (None, [i32, i32, vp, vp, vp, pd]),
    "h264_deblock_picture_structure": (None, [i32]),
    "h264_deblock_chroma422": (None, [vp]),
    "h264_deblock_params": (i32, [i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, i32, i32, vp]),
    "h264_deblock_params_hbd": (i32, [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, i32, i32, vp]),
    "h264_deblock_picture_with": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, i32, i32]),
    "h264_deblock_picture_with_hbd": (i32, [i32, vp, vp, vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, i32, i32]),
    "h264_pictures": (i32, [vp, vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32]),
    "me_cmp_select": (None, [vp, i32, vp]),
    "table_fill": (i32, [i32, i32, i32, vp, i32]),
    "pred_table_fill": (i32, [i32, i32, vp, i32]),
    "mpeg_dequant": (None, [i32, vp, i32, i32, i32, i32, i32, vp, vp, i32, i32, i32]),
    "mpeg_scantables": (None, [i32, vp, vp]),
    "me_cmp_quant": (i32, [i32, i32, vp, vp, vp, pd, i32, vp]),
    "enc_qmatrices": (None, [vp, vp, vp, vp]),
    "h264_pred": (None, [i32, i32, vp, vp, i32, i32, pd]),
    "h264_pred_add": (None, [i32, i32, vp, vp, vp, i32, i32, pd]),
    "mpeg4_qpel": (None, [i32, i32, i32, vp, vp, pd]),
    "pixblock": (None, [i32, vp, vp, vp, pd]),
    "h264_weight": (None, [i32, vp, i32, i32, i32, i32, i32]),
    "h264_biweight": (None, [i32, vp, vp, i32, i32, i32, i32, i32, i32]),
    "h264_add_pixels_clear": (None, [i32, vp, vp, i32]),
    "h264_qpel": (None, [i32, i32, i32, vp, vp, pd]),
    "h264_chroma": (None, [i32, i32, vp, vp, pd, i32, i32, i32]),
    "hpel": (i32, [i32, i32, i32, vp, vp, pd, i32]),
    "me_cmp": (i32, [i32, i32, i32, vp, vp, pd, i32]),
    "full_search": (None, [vp, vp, i32, i32, i32, i32, i32, i32, vp, i32]),
    "sws_yuv420p_to_rgb24": (i32, [vp, vp, i32, i32, vp, i32, i32, i32, i32]),
    "sws_yuv420p_to_yuv420p": (i32, [vp, vp, i32, i32, vp, vp, i32, i32, i32]),
    "sws_set_colorspace": (None, [vp, i32, i32, i32, i32]),
    "sws_planar": (i32, [i32, vp, vp, i32, i32, i32, vp, vp, i32, i32, i32]),
    "sws_nv12": (i32, [i32, vp, i32, vp, i32, i32, i32, i32, vp, vp, i32, i32, i32]),
    "sws_set_filter": (None, [i32, i32, vp, i32]),
    "sws_line_range": (i32, [i32, vp, vp, i32]),
    "sws_line_hscale": (i32, [i32, i32, vp, i32, vp, vp, vp, i32]),
    "sws_line_hfast": (i32, [i32, vp, vp, i32, vp, vp, i32, i32]),
    "sws_line_plane": (i32, [i32, vp, i32, vp, vp, i32, vp, i32]),
    "sws_line_nv12": (i32, [i32, vp, i32, vp, vp, vp, i32]),
    "sws_line_packed": (i32, [i32, i32, i32, vp, vp, i32, vp, vp, vp, i32, vp, i32, i32, i32, i32]),
    "sws_open": (vp, [i32, i32, i32, i32, i32, i32, i32]),
    "sws_set_slots": (i32, [vp, vp]),
    "sws_slot_mask": (i32, [vp]),
    "sws_run": (i32, [vp, vp, vp, i32, vp, vp]),
    "sws_run_slice": (i32, [vp, vp, vp, i32, i32, vp, vp]),
    "sws_close": (None, [vp]),
    "sws_get_filter": (i32, [i32, i32, i32, i32, i32, i32, i32, vp, vp, i32, vp]),
    "sws_rgb24_tables": (None, [vp, vp, vp, vp, vp]),
    "fft": (None, [i32, i32, vp]),
    "imdct_half": (None, [i32, dbl, vp, vp]),
    "imdct_calc": (None, [i32, dbl, vp, vp]),
    "mdct_calc": (None, [i32, dbl, vp, vp]),
}


class Oracle:
    def __init__(self, path, prefix):
        self.path, self.prefix = path, prefix
        self.lib = C.CDLL(path)
        self.missing = []
        for name, (res, args) in API.items():
            try:
                f = getattr(self.lib, prefix + name)
            except AttributeError:
                self.missing.append(name)
                continue
            f.restype, f.argtypes = res, args
            setattr(self, name, f)

    def has(self, name):
        return hasattr(self, name)


_cache = {}


def port():
    if "port" not in _cache:
        if not os.path.exists(PORT_PATH):
            raise RuntimeError("oracle port not built: run __graft_entry__.build()")
        _cache["port"] = Oracle(PORT_PATH, "orc_")
    return _cache["port"]


def ref():
    """The compiled reference, or None when oracle/_ref has not been built (no /root/reference)."""
    if "ref" not in _cache:
        _cache["ref"] = Oracle(REF_PATH, "ref_") if os.path.exists(REF_PATH) else None
    return _cache["ref"]


def ref_lib(name):
    """The satellite library oracle/_ref/lib<name>ref.so (one feature of the unmodified reference, linked against libavref.so), or None
    when it has not been built."""
    key = "lib" + name
    if key not in _cache:
        path = os.path.join(_HERE, "_ref", "lib%sref.so" % name)
        _cache[key] = C.CDLL(path) if os.path.exists(path) else None
    return _cache[key]


def ref_simd():
    """TIMING ONLY: the same unmodified reference sources configured the way its own configure does on this x86-64 host without an
    external assembler (ARCH_X86, inline-asm MMX / SSE2 / SSSE3 on, cpu flags unmasked, idct_algo FF_IDCT_AUTO) -- bench.py's
    "x86 SIMD" CPU figure.  Never a parity oracle (the MMX IDCT is a different algorithm).  None when it has not been built."""
    if "ref_simd" not in _cache:
        _cache["ref_simd"] = Oracle(REF_SIMD_PATH, "ref_") if os.path.exists(REF_SIMD_PATH) else None
    return _cache["ref_simd"]


def ptr(a):
    """numpy array -> void* (array must stay alive)."""
    return a.ctypes.data_as(vp)
