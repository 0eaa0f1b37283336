"""ctypes mirrors of the reference's DSP function-pointer tables (include/avdsp_b200_tables.h), so the harness
can call the slots that ff_*_init_cuda() installs exactly the way a codec calls them."""
import ctypes as C

u8p, i16p, i8p = C.POINTER(C.c_uint8), C.POINTER(C.c_int16), C.POINTER(C.c_int8)
pd = C.c_ssize_t
FF_IDCT_AUTO, FF_IDCT_SIMPLE, FF_IDCT_XVID = 0, 2, 14

_clamped = C.CFUNCTYPE(None, i16p, u8p, pd)
_idct = C.CFUNCTYPE(None, i16p)
_idct_px = C.CFUNCTYPE(None, u8p, pd, i16p)


class IDCTDSPContext(C.Structure):          # libavcodec/idctdsp.h:53-98
    _fields_ = [("put_pixels_clamped", _clamped), ("put_signed_pixels_clamped", _clamped), ("add_pixels_clamped", _clamped),
                ("idct", _idct), ("idct_put", _idct_px), ("idct_add", _idct_px),
                ("idct_permutation", C.c_uint8 * 64), ("perm_type", C.c_int)]


class ProresDSPContext(C.Structure):        # libavcodec/proresdsp.h:31-35
    _fields_ = [("idct_permutation_type", C.c_int), ("idct_permutation", C.c_uint8 * 64),
                ("idct_put", C.CFUNCTYPE(None, C.POINTER(C.c_uint16), pd, i16p, i16p))]


class FFProresSlice(C.Structure):           # include/avdsp_b200.h
    _fields_ = [("first_block", C.c_uint32), ("sf", C.c_uint16), ("reserved", C.c_uint16)]


class FFProresPictureWork(C.Structure):     # include/avdsp_b200.h
    _fields_ = [("data", C.c_void_p * 3), ("linesize", C.c_int * 3), ("mb_rows", C.c_int * 3), ("mb_width", C.c_int),
                ("mb_height", C.c_int), ("slice_width_factor", C.c_int), ("chroma_format", C.c_int),
                ("qmat_luma", C.c_uint8 * 64), ("qmat_chroma", C.c_uint8 * 64), ("slices", C.c_void_p), ("n_slices", C.c_int),
                ("blocks", C.c_void_p), ("n_blocks", C.c_size_t)]


class FFProresFrameInfo(C.Structure):       # include/avdsp_b200.h
    _fields_ = [("pix_fmt", C.c_int), ("interlaced_frame", C.c_int), ("top_field_first", C.c_int), ("color_primaries", C.c_int),
                ("color_trc", C.c_int), ("colorspace", C.c_int), ("lines", C.c_int), ("pictures", C.c_int), ("result", C.c_int)]


class FFProresDecodeWork(C.Structure):      # include/avdsp_b200.h
    _fields_ = [("pkt_host", C.c_void_p), ("pkt", C.c_void_p), ("size", C.c_int), ("width", C.c_int), ("height", C.c_int),
                ("data", C.c_void_p * 4), ("linesize", C.c_int * 4), ("lines", C.c_int * 4)]


class FFProresEncodeWork(C.Structure):      # include/avdsp_b200.h
    _fields_ = [("data", C.c_void_p * 4), ("linesize", C.c_int * 4), ("width", C.c_int), ("height", C.c_int), ("pix_fmt", C.c_int),
                ("interlaced", C.c_int), ("profile", C.c_int), ("mbs_per_slice", C.c_int), ("bits_per_mb", C.c_int),
                ("quant_sel", C.c_int), ("alpha_bits", C.c_int), ("force_quant", C.c_int), ("vendor", C.c_char * 4),
                ("color_primaries", C.c_uint8), ("color_trc", C.c_uint8), ("colorspace", C.c_uint8), ("out", C.c_void_p),
                ("out_capacity", C.c_size_t), ("out_size", C.c_void_p)]


class FFDnxhdCidEntry(C.Structure):         # include/avdsp_b200.h (CIDEntry, libavcodec/dnxhddata.h:28-42)
    _fields_ = [("cid", C.c_int), ("width", C.c_uint), ("height", C.c_uint), ("interlaced", C.c_int), ("frame_size", C.c_uint),
                ("coding_unit_size", C.c_uint), ("index_bits", C.c_int), ("bit_depth", C.c_int),
                ("luma_weight", C.c_void_p), ("chroma_weight", C.c_void_p), ("dc_codes", C.c_void_p), ("dc_bits", C.c_void_p),
                ("ac_codes", C.c_void_p), ("ac_bits", C.c_void_p), ("ac_level", C.c_void_p), ("ac_run_flag", C.c_void_p),
                ("ac_index_flag", C.c_void_p), ("run_codes", C.c_void_p), ("run_bits", C.c_void_p), ("run", C.c_void_p),
                ("bit_rates", C.c_int * 5)]


class FFDnxhdRcState(C.Structure):          # include/avdsp_b200.h
    _fields_ = [("qscale", C.c_uint32), ("lambda_", C.c_uint32)]


class FFDnxhdEncodeWork(C.Structure):       # include/avdsp_b200.h
    _fields_ = [("data", C.c_void_p * 3), ("linesize", C.c_int * 3), ("cid_table", C.c_void_p), ("interlaced", C.c_int),
                ("dct_algo", C.c_int), ("mb_decision", C.c_int), ("qmax", C.c_int), ("nitris_compat", C.c_int), ("state", C.c_void_p),
                ("out", C.c_void_p), ("out_capacity", C.c_size_t), ("out_info", C.c_void_p)]


class FFDnxhdFrameInfo(C.Structure):        # include/avdsp_b200.h
    _fields_ = [("cid", C.c_int), ("width", C.c_int), ("height", C.c_int), ("pix_fmt", C.c_int), ("interlaced_frame", C.c_int),
                ("top_field_first", C.c_int), ("sar_num", C.c_int), ("sar_den", C.c_int), ("lines", C.c_int)]


class FFDnxhdDecodeWork(C.Structure):       # include/avdsp_b200.h
    _fields_ = [("pkt_host", C.c_void_p), ("pkt", C.c_void_p), ("size", C.c_int), ("data", C.c_void_p * 3), ("linesize", C.c_int * 3),
                ("lines", C.c_int * 3), ("gray", C.c_int)]


class FDCTDSPContext(C.Structure):          # libavcodec/fdctdsp.h:26-29
    _fields_ = [("fdct", _idct), ("fdct248", _idct)]


_fill = C.CFUNCTYPE(None, u8p, C.c_uint8, pd, C.c_int)


class BlockDSPContext(C.Structure):         # libavcodec/blockdsp.h:32-37
    _fields_ = [("clear_block", _idct), ("clear_blocks", _idct), ("fill_block_tab", _fill * 2)]


me_cmp_func = C.CFUNCTYPE(C.c_int, C.c_void_p, u8p, u8p, pd, C.c_int)


class MECmpContext(C.Structure):            # libavcodec/me_cmp.h:39-63
    _fields_ = [("sum_abs_dctelem", C.CFUNCTYPE(C.c_int, i16p))] + \
        [(n, me_cmp_func * 6) for n in ("sad", "sse", "hadamard8_diff", "dct_sad", "quant_psnr", "bit", "rd", "vsad", "vsse", "nsse",
                                         "dct_max", "dct264_sad", "me_pre_cmp", "me_cmp", "me_sub_cmp", "mb_cmp", "ildct_cmp",
                                         "frame_skip_cmp")] + [("pix_abs", (me_cmp_func * 4) * 2)]


_weight = C.CFUNCTYPE(None, u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)
_biweight = C.CFUNCTYPE(None, u8p, u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)
_lf = C.CFUNCTYPE(None, u8p, C.c_int, C.c_int, C.c_int, i8p)
_lfi = C.CFUNCTYPE(None, u8p, C.c_int, C.c_int, C.c_int)
_hidct = C.CFUNCTYPE(None, u8p, i16p, C.c_int)
_hidct_mb = C.CFUNCTYPE(None, u8p, C.POINTER(C.c_int), i16p, C.c_int, u8p)
_hidct_mb8 = C.CFUNCTYPE(None, C.POINTER(u8p), C.POINTER(C.c_int), i16p, C.c_int, u8p)


class H264DSPContext(C.Structure):          # libavcodec/h264dsp.h:41-117
    _fields_ = [("weight_h264_pixels_tab", _weight * 4), ("biweight_h264_pixels_tab", _biweight * 4),
                ("h264_v_loop_filter_luma", _lf), ("h264_h_loop_filter_luma", _lf), ("h264_h_loop_filter_luma_mbaff", _lf),
                ("h264_v_loop_filter_luma_intra", _lfi), ("h264_h_loop_filter_luma_intra", _lfi), ("h264_h_loop_filter_luma_mbaff_intra", _lfi),
                ("h264_v_loop_filter_chroma", _lf), ("h264_h_loop_filter_chroma", _lf), ("h264_h_loop_filter_chroma_mbaff", _lf),
                ("h264_v_loop_filter_chroma_intra", _lfi), ("h264_h_loop_filter_chroma_intra", _lfi), ("h264_h_loop_filter_chroma_mbaff_intra", _lfi),
                ("h264_loop_filter_strength", C.c_void_p),
                ("h264_idct_add", _hidct), ("h264_idct8_add", _hidct), ("h264_idct_dc_add", _hidct), ("h264_idct8_dc_add", _hidct),
                ("h264_idct_add16", _hidct_mb), ("h264_idct8_add4", _hidct_mb), ("h264_idct_add8", _hidct_mb8), ("h264_idct_add16intra", _hidct_mb),
                ("h264_luma_dc_dequant_idct", C.CFUNCTYPE(None, i16p, i16p, C.c_int)),
                ("h264_chroma_dc_dequant_idct", C.CFUNCTYPE(None, i16p, C.c_int)),
                ("h264_add_pixels8_clear", _hidct), ("h264_add_pixels4_clear", _hidct),
                ("startcode_find_candidate", C.CFUNCTYPE(C.c_int, u8p, C.c_int))]


h263_loop_filter_func = C.CFUNCTYPE(None, u8p, C.c_int, C.c_int)


class H263DSPContext(C.Structure):          # libavcodec/h263dsp.h:26-29
    _fields_ = [("h263_h_loop_filter", h263_loop_filter_func), ("h263_v_loop_filter", h263_loop_filter_func)]


gmc1_func = C.CFUNCTYPE(None, u8p, u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)
gmc_func = C.CFUNCTYPE(None, u8p, u8p, *([C.c_int] * 12))


class MpegVideoDSPContext(C.Structure):     # libavcodec/mpegvideodsp.h:27-41
    _fields_ = [("gmc1", gmc1_func), ("gmc", gmc_func)]


qpel_mc_func = C.CFUNCTYPE(None, u8p, u8p, pd)


class H264QpelContext(C.Structure):         # libavcodec/h264qpel.h:27-30
    _fields_ = [("put_h264_qpel_pixels_tab", (qpel_mc_func * 16) * 4), ("avg_h264_qpel_pixels_tab", (qpel_mc_func * 16) * 4)]


h264_chroma_mc_func = C.CFUNCTYPE(None, u8p, u8p, pd, C.c_int, C.c_int, C.c_int)


class H264ChromaContext(C.Structure):       # libavcodec/h264chroma.h:25-30
    _fields_ = [("put_h264_chroma_pixels_tab", h264_chroma_mc_func * 3), ("avg_h264_chroma_pixels_tab", h264_chroma_mc_func * 3)]


op_pixels_func = C.CFUNCTYPE(None, u8p, u8p, pd, C.c_int)


class HpelDSPContext(C.Structure):          # libavcodec/hpeldsp.h:45-93
    _fields_ = [("put_pixels_tab", (op_pixels_func * 4) * 4), ("avg_pixels_tab", (op_pixels_func * 4) * 4),
                ("put_no_rnd_pixels_tab", (op_pixels_func * 4) * 4), ("avg_no_rnd_pixels_tab", op_pixels_func * 4)]


class FFTContext(C.Structure):              # libavcodec/fft.h:73-99
    pass


_fftc = C.CFUNCTYPE(None, C.POINTER(FFTContext), C.c_void_p)
_mdctf = C.CFUNCTYPE(None, C.POINTER(FFTContext), C.POINTER(C.c_float), C.POINTER(C.c_float))
FFTContext._fields_ = [("nbits", C.c_int), ("inverse", C.c_int), ("revtab", C.POINTER(C.c_uint16)), ("tmp_buf", C.c_void_p),
                       ("mdct_size", C.c_int), ("mdct_bits", C.c_int), ("tcos", C.POINTER(C.c_float)), ("tsin", C.POINTER(C.c_float)),
                       ("fft_permute", _fftc), ("fft_calc", _fftc), ("imdct_calc", _mdctf), ("imdct_half", _mdctf), ("mdct_calc", _mdctf),
                       ("mdct_calcw", C.c_void_p), ("fft_permutation", C.c_int), ("mdct_permutation", C.c_int)]


class FFH264DeblockSlice(C.Structure):
    """include/avdsp_b200.h FFH264DeblockSlice (133 int32)"""
    _fields_ = [("alpha_c0_offset", C.c_int32), ("beta_offset", C.c_int32), ("deblocking_filter", C.c_int32),
                ("list_count", C.c_int32), ("qp_thresh", C.c_int32), ("ref2frm", (C.c_int32 * 64) * 2)]


class FFH264DeblockInfo(C.Structure):
    """include/avdsp_b200.h FFH264DeblockInfo (host struct holding device pointers)"""
    _fields_ = [("mb_w", C.c_int), ("mb_h", C.c_int), ("n_pictures", C.c_int),
                ("mb_type", C.c_void_p), ("qscale_table", C.c_void_p), ("non_zero_count", C.c_void_p),
                ("cbp_table", C.c_void_p), ("slice_table", C.c_void_p),
                ("motion_val", C.c_void_p * 2), ("ref_index", C.c_void_p * 2),
                ("slices", C.c_void_p), ("n_slices", C.c_int), ("chroma_qp_table", C.c_void_p),
                ("cabac", C.c_int), ("transform_8x8_mode", C.c_int), ("field_picture", C.c_int), ("chroma422", C.c_void_p)]


class FFH264PictureWork(C.Structure):
    """include/avdsp_b200.h FFH264PictureWork (host struct holding device pointers): ff_h264_flush_pictures_cuda"""
    _fields_ = [("mb_w", C.c_int), ("mb_h", C.c_int), ("n_pictures", C.c_int),
                ("luma", C.c_void_p), ("cb", C.c_void_p), ("cr", C.c_void_p), ("linesize", C.c_int), ("uvlinesize", C.c_int),
                ("mc", C.c_void_p), ("n_mc", C.c_size_t), ("refs", C.c_void_p),
                ("weight", C.c_void_p * 3), ("n_weight", C.c_size_t * 3), ("weight_src", C.c_void_p * 3),
                ("coeffs", C.c_void_p), ("coeff_stride", C.c_size_t), ("nnzc", C.c_void_p),
                ("dc", C.c_void_p), ("luma_dc", C.c_void_p), ("residual", C.c_void_p), ("intra", C.c_void_p),
                ("deblock_info", C.POINTER(FFH264DeblockInfo)), ("deblock_records", C.c_void_p), ("progress", C.c_void_p),
                ("bit_depth", C.c_int), ("chroma_format_idc", C.c_int), ("deblock_chroma422", C.c_void_p)]


class FFMpegDequantTables(C.Structure):
    """include/avdsp_b200.h FFMpegDequantTables"""
    _fields_ = [("intra_matrix", C.c_uint16 * 64), ("inter_matrix", C.c_uint16 * 64), ("permutated", C.c_uint8 * 64),
                ("raster_end", C.c_uint8 * 64), ("alternate_scan", C.c_int), ("h263_aic", C.c_int)]


class FFMpvMCPicture(C.Structure):
    """include/avdsp_b200.h FFMpvMCPicture (host struct holding device pointers): ff_mpv_motion_batch_cuda"""
    _fields_ = [("dest", C.c_void_p * 3), ("cur", C.c_void_p * 3), ("last", C.c_void_p * 3), ("next", C.c_void_p * 3),
                ("linesize", C.c_int), ("uvlinesize", C.c_int), ("pic_linesize", C.c_int), ("pic_uvlinesize", C.c_int),
                ("mb_width", C.c_int), ("mb_height", C.c_int), ("width", C.c_int), ("height", C.c_int),
                ("h_edge_pos", C.c_int), ("v_edge_pos", C.c_int), ("out_format", C.c_int), ("picture_structure", C.c_int),
                ("first_field", C.c_int), ("b_picture", C.c_int), ("no_rounding", C.c_int), ("quarter_sample", C.c_int),
                ("workaround_bugs", C.c_int), ("chroma_format", C.c_int), ("obmc", C.c_int), ("sprite", C.c_int), ("mspel", C.c_int),
                ("lowres", C.c_int), ("recs", C.c_void_p), ("n_recs", C.c_size_t), ("obmc_recs", C.c_void_p),
                ("sprite_warping_accuracy", C.c_int), ("real_sprite_warping_points", C.c_int),
                ("sprite_offset", (C.c_int * 2) * 2), ("sprite_delta", (C.c_int * 2) * 2), ("interlaced", C.c_int)]


class FFMpvResidualBatch(C.Structure):
    """include/avdsp_b200.h FFMpvResidualBatch: one residual stage of ff_mpv_flush_pictures_cuda"""
    _fields_ = [("transform", C.c_int), ("dequant", C.c_int), ("mode", C.c_int), ("tables", C.c_void_p), ("recs", C.c_void_p),
                ("blocks", C.c_void_p), ("frame", C.c_void_p), ("dst_off", C.c_void_p), ("stride", C.c_ssize_t), ("n", C.c_size_t),
                ("clear", C.c_int)]


class FFH263LoopFilterPicture(C.Structure):
    """include/avdsp_b200.h FFH263LoopFilterPicture (host struct holding device pointers): ff_h263_loop_filter_batch_cuda"""
    _fields_ = [("data", C.c_void_p * 3), ("linesize", C.c_int), ("uvlinesize", C.c_int), ("mb_width", C.c_int), ("mb_height", C.c_int),
                ("mb_stride", C.c_int), ("mb_type", C.c_void_p), ("qscale_table", C.c_void_p), ("chroma_qscale_table", C.c_uint8 * 32)]


class FFMpvPictureWork(C.Structure):
    """include/avdsp_b200.h FFMpvPictureWork (host struct): ff_mpv_flush_pictures_cuda"""
    _fields_ = [("pictures", C.c_void_p), ("n_pictures", C.c_int), ("rejected", C.c_void_p),
                ("residual", C.c_void_p), ("n_residual", C.c_int), ("loop_filter", C.c_void_p), ("n_loop_filter", C.c_int)]


class FFMECmpEncState(C.Structure):
    """include/avdsp_b200.h FFMECmpEncState: the MpegEncContext fields quant_psnr / bit / rd read (me_cmp.c:621-782)"""
    _fields_ = [("fdct", C.c_int32), ("dequant", C.c_int32), ("qscale", C.c_int32), ("mb_intra", C.c_int32), ("y_dc_scale", C.c_int32),
                ("h263_aic", C.c_int32), ("intra_quant_bias", C.c_int32), ("inter_quant_bias", C.c_int32), ("ac_esc_length", C.c_int32),
                ("q_intra_matrix", C.c_int32 * 64), ("q_inter_matrix", C.c_int32 * 64), ("intra_matrix", C.c_uint16 * 64),
                ("inter_matrix", C.c_uint16 * 64), ("scantable", C.c_uint8 * 64)]


class FFMECmpVlcTables(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("intra_ac_vlc_length", "intra_ac_vlc_last_length", "inter_ac_vlc_length", "inter_ac_vlc_last_length",
                                          "luma_dc_vlc_length")]


class FFMECmpEncView(C.Structure):
    """include/avdsp_b200.h FFMECmpEncView: host pointers into a live MpegEncContext"""
    _fields_ = [(n, C.c_void_p) for n in ("qscale", "y_dc_scale", "h263_aic", "intra_quant_bias", "inter_quant_bias", "ac_esc_length", "mb_intra",
                                          "block_last_index", "q_intra_matrix", "q_inter_matrix", "intra_matrix", "inter_matrix", "scantable",
                                          "intra_ac_vlc_length", "intra_ac_vlc_last_length", "inter_ac_vlc_length", "inter_ac_vlc_last_length",
                                          "luma_dc_vlc_length")] + \
        [(n, C.c_int) for n in ("fdct", "dequant", "idct_perm_none", "plain_quantiser")]


class FFMpvQuantState(C.Structure):
    """include/avdsp_b200.h FFMpvQuantState: the MpegEncContext fields the encoder's quantisers read that stay fixed over a picture"""
    _fields_ = [(n, C.c_int32) for n in ("fdct", "out_format", "mpeg_quant", "h263_aic", "intra_quant_bias", "inter_quant_bias", "ac_esc_length",
                                         "min_qcoeff", "max_qcoeff", "luma_elim_threshold", "chroma_elim_threshold")] + \
        [("q_intra_matrix", (C.c_int32 * 64) * 32), ("q_inter_matrix", (C.c_int32 * 64) * 32), ("intra_matrix", C.c_uint16 * 64),
         ("inter_matrix", C.c_uint16 * 64), ("scantable", C.c_uint8 * 64), ("pad", C.c_uint8 * 8)]


class FFMpvQuantRecord(C.Structure):
    """include/avdsp_b200.h FFMpvQuantRecord (8 bytes, one per block)"""
    _fields_ = [("qscale", C.c_uint8), ("intra", C.c_uint8), ("dc_scale", C.c_uint8), ("chroma", C.c_uint8), ("lambda2", C.c_uint32)]


class FFMpvNoiseReduction(C.Structure):
    """include/avdsp_b200.h FFMpvNoiseReduction: device pointers to dct_offset [2][64], dct_error_sum [2][64], dct_count [2]"""
    _fields_ = [("dct_offset", C.c_void_p), ("dct_error_sum", C.c_void_p), ("dct_count", C.c_void_p)]


class FFMpvQuantView(C.Structure):
    """include/avdsp_b200.h FFMpvQuantView: host pointers into a live MpegEncContext"""
    _fields_ = [(n, C.c_void_p) for n in ("mb_intra", "y_dc_scale", "c_dc_scale", "h263_aic", "lambda2", "intra_quant_bias", "inter_quant_bias",
                                          "ac_esc_length", "min_qcoeff", "max_qcoeff", "q_intra_matrix", "q_inter_matrix", "intra_matrix",
                                          "inter_matrix", "scantable", "intra_ac_vlc_length", "intra_ac_vlc_last_length", "inter_ac_vlc_length",
                                          "inter_ac_vlc_last_length", "dct_error_sum", "dct_offset", "dct_count", "coded_score",
                                          "dct_quantize", "fast_dct_quantize")] + \
        [(n, C.c_int) for n in ("fdct", "out_format", "mpeg_quant", "idct_perm_none", "quantizer_noise_shaping", "slice_context_count")]


# the reference's s->dct_quantize signature (mpegvideo.h:499)
DCT_QUANTIZE_FUNC = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int))


_p4 = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t)
_p8l = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.c_ssize_t)
_p8 = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t)
_pa = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t)
_pfa = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_ssize_t)
_pba = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t)


class H264PredContext(C.Structure):         # libavcodec/h264pred.h:91-110
    _fields_ = [("pred4x4", _p4 * 15), ("pred8x8l", _p8l * 12), ("pred8x8", _p8 * 11), ("pred16x16", _p8 * 9),
                ("pred4x4_add", _pa * 2), ("pred8x8l_add", _pa * 2), ("pred8x8l_filter_add", _pfa * 2),
                ("pred8x8_add", _pba * 3), ("pred16x16_add", _pba * 3)]


class PixblockDSPContext(C.Structure):      # libavcodec/pixblockdsp.h:27-35
    _fields_ = [("get_pixels", C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t)),
                ("diff_pixels", C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t))]


class QpelDSPContext(C.Structure):          # libavcodec/qpeldsp.h:69-73
    _fields_ = [("put_qpel_pixels_tab", (qpel_mc_func * 16) * 2), ("avg_qpel_pixels_tab", (qpel_mc_func * 16) * 2),
                ("put_no_rnd_qpel_pixels_tab", (qpel_mc_func * 16) * 2)]


_vp, _i = C.c_void_p, C.c_int


class SwsLineSlotsCUDA(C.Structure):        # include/avdsp_b200.h SwsLineSlotsCUDA: the SwsContext per-line slots (swscale_internal.h:312-330,478-535)
    _fields_ = [("hyScale", C.CFUNCTYPE(None, _vp, _vp, _i, _vp, _vp, _vp, _i)), ("hcScale", C.CFUNCTYPE(None, _vp, _vp, _i, _vp, _vp, _vp, _i)),
                ("hyscale_fast", C.CFUNCTYPE(None, _vp, _vp, _i, _vp, _i, _i)), ("hcscale_fast", C.CFUNCTYPE(None, _vp, _vp, _vp, _i, _vp, _vp, _i, _i)),
                ("yuv2plane1", C.CFUNCTYPE(None, _vp, _vp, _i, _vp, _i)), ("yuv2planeX", C.CFUNCTYPE(None, _vp, _i, _vp, _vp, _i, _vp, _i)),
                ("yuv2nv12cX", C.CFUNCTYPE(None, _vp, _vp, _i, _vp, _vp, _vp, _i)),
                ("yuv2packed1", C.CFUNCTYPE(None, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i)),
                ("yuv2packed2", C.CFUNCTYPE(None, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i)),
                ("yuv2packedX", C.CFUNCTYPE(None, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _i, _i)),
                ("lumConvertRange", C.CFUNCTYPE(None, _vp, _i)), ("chrConvertRange", C.CFUNCTYPE(None, _vp, _vp, _i))]
