"""CPU: the product's H.264 slot path (libav_b200/csrc/slots.cu + h264dsp.cuh: staging, argument packing, the per-call slot
kernel, the table hooks) compiled unchanged as host C++ (tests/hostsim/) and driven through the same cases as the GPU tests
(tests/slot_cases.py), against the oracle.  Not the product and not a fallback: tests/hostsim/libhostsim.so is only ever
loaded by the CPU suite.  The GPU tests remain the parity tests proper; this keeps the slot code checked while it changes without a GPU."""
import ctypes as C

import numpy as np
import pytest

import hostsim_build
import slot_cases


@pytest.fixture
def sim(built):
    return hostsim_build.fresh()


def last_error_of(lib):
    return lambda: lib.avb200_last_error().decode()


def test_h264_qpel_and_chroma_slots(sim, checker):
    slot_cases.qpel_and_chroma_cases(sim, last_error_of(sim), checker)


def test_h264dsp_slots(sim, checker):
    slot_cases.h264dsp_cases(sim, last_error_of(sim), checker, weights=False)


def test_startcode_slot(sim):
    import numpy as np
    from libav_b200 import tables
    for bits in (8, 10):
        c = tables.H264DSPContext()
        sim.ff_h264dsp_init_cuda(C.byref(c), bits, 1)
        slot_cases.startcode_cases(np.random.default_rng(bits), c.startcode_find_candidate)
    assert sim.avb200_last_error().decode() == ""


def test_h264dsp_slots_422(sim, checker):
    slot_cases.h264dsp_422_cases(sim, last_error_of(sim), checker)


def test_batched_kernels_are_not_simulated(sim):
    from libav_b200 import tables
    c = tables.H264DSPContext()
    sim.ff_h264dsp_init_cuda(C.byref(c), 8, 1)
    import numpy as np
    pix = np.zeros((16, 32), np.uint8)
    c.weight_h264_pixels_tab[0](slot_cases.P(pix), 32, 8, 5, 37, -3)
    assert "not simulated" in sim.avb200_last_error().decode()
    sim.avb200_clear_error()


def test_sws_line_slots(sim, refo):
    """libswscale's per-line slots (libav_b200/csrc/sws_slots.cu, host-compiled) against the functions the compiled reference installs; the
    contexts come from the host-compiled sws_getContext_cuda() (swscale_hostsim.cpp)"""
    import sws_line_cases as L

    def run(colourspace):
        def make_ctx(dst_fmt, flags, src_fmt=0):
            ctx = sim.sws_getContext_cuda(64, 48, src_fmt, 96, 80, dst_fmt, flags, None, None, None)
            assert ctx, (dst_fmt, flags, sim.avb200_last_error())
            if colourspace and dst_fmt in L.PACKED_FMTS and dst_fmt not in (1, 15):
                tab = (C.c_int * 4)(*colourspace[0])
                assert sim.sws_setColorspaceDetails_cuda(ctx, tab, colourspace[1], tab, 0, *colourspace[2:]) == 0
            return ctx, sim.sws_freeContext_cuda
        calls = L.SlotCalls(sim, make_ctx, last_error_of(sim))
        try:
            return L.compare(calls, L.OracleCalls(refo), seed=3 if colourspace else 4)
        finally:
            calls.close()
    assert run(None) > 150
    refo.sws_set_colorspace((C.c_int * 4)(*L.FCC), 0, 3000, 70000, 60000)
    try:
        assert run((L.FCC, 0, 3000, 70000, 60000)) > 150
    finally:
        refo.sws_set_colorspace(None, 0, 0, 0, 0)
    assert sim.avb200_last_error().decode() == ""


def test_sws_line_slot_registration(sim):
    """a slot called for a SwsContext that was never registered (or whose SwsContextCUDA was freed) fails loudly"""
    import numpy as np
    import sws_line_cases as L
    from libav_b200 import tables
    t = tables.SwsLineSlotsCUDA()
    assert sim.ff_sws_init_swscale_cuda(None, None, C.byref(t)) == -1
    sim.avb200_clear_error()
    ctx = sim.sws_getContext_cuda(64, 48, 0, 96, 80, 2, 4, None, None, None)
    assert sim.ff_sws_init_swscale_cuda(C.c_void_p(0x7000), C.c_void_p(ctx), C.byref(t)) == 0
    sim.sws_freeContext_cuda(ctx)
    lum, cu, out = np.zeros(64, np.int16), np.zeros(64, np.int16), np.full(256, 9, np.uint8)
    t.yuv2packed1(C.c_void_p(0x7000), L.vp(lum), L.ptrs([cu, cu]), L.ptrs([cu, cu]), None, L.vp(out), 16, 0, 0)
    assert "not registered" in sim.avb200_last_error().decode() and (out == 9).all()
    sim.avb200_clear_error()


@pytest.mark.parametrize("bits", [9, 10])
def test_h264_high_bit_depth_slots(sim, refo, bits):
    """the 9 / 10-bit instances of H264DSPContext / H264QpelContext / H264ChromaContext / H264PredContext (libav_b200/csrc/slots_hbd.cu,
    h264pred_hbd.cu, host-compiled) against
    the tables the compiled reference fills for those depths"""
    import hbd_cases
    assert hbd_cases.compare(hbd_cases.TableCallee(sim, pred_init=sim.hostsim_h264_pred_init_hbd), refo, bits, seed=2) > 800
    assert sim.avb200_last_error().decode() == ""


def test_simple_idct10(sim, refo):
    """the 10-bit simple IDCT (libav_b200/csrc/idct10.cu, host-compiled): the three table entries and the batched entry point"""
    import numpy as np
    import idct10_cases
    from libav_b200 import tables
    t = tables.IDCTDSPContext()
    sim.hostsim_idctdsp_init10(C.byref(t))
    assert idct10_cases.slot_cases(t, refo) == 360
    sim.ff_simple_idct10_batch_cuda.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_size_t, C.c_void_p]

    def run_batch(mode, blk, frame, off):          # host simulation: "device memory" is host memory
        assert sim.ff_simple_idct10_batch_cuda(mode, blk.ctypes.data, frame.ctypes.data, off.ctypes.data, frame.strides[0], len(blk), None) == 0
        return blk, frame
    for mode in range(3):
        idct10_cases.batch_case(run_batch, refo, mode)
        idct10_cases.batch_case(run_batch, refo, mode, n=1003, pad=8)
        idct10_cases.batch_case(run_batch, refo, mode, n=1000, pad=8, shift=1, seed=7)
    assert sim.ff_simple_idct10_batch_cuda(3, None, None, None, 0, 0, None) == -1
    sim.avb200_clear_error()


def test_fdct10(sim, refo):
    """ff_fdctdsp_init_cuda(c, dct_algo, 10, 1): the 10-bit accurate forward DCT pair (libav_b200/csrc/fdct10.cu through slots.cu, host-compiled)"""
    import idct10_cases
    from libav_b200 import tables
    t = tables.FDCTDSPContext()
    sim.ff_fdctdsp_init_cuda(C.byref(t), 0, 10, 1)
    sim.ff_fdct_batch_cuda.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]

    def run_batch(which, blk):
        assert sim.ff_fdct_batch_cuda(which, blk.ctypes.data, len(blk), None) == 0
        return blk
    idct10_cases.fdct10_cases(t, run_batch, refo)
    assert sim.avb200_last_error().decode() == ""


def _enc_protos(lib):
    lib.ff_me_cmp_enc_state_cuda.restype = C.c_void_p
    lib.ff_me_cmp_enc_state_cuda.argtypes = [C.c_void_p, C.c_void_p]
    lib.ff_me_cmp_enc_state_free_cuda.argtypes = [C.c_void_p]
    lib.ff_me_cmp_enc_batch_cuda.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ff_me_cmp_enc_init_cuda.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ff_me_cmp_enc_uninit_cuda.argtypes = [C.c_void_p]


def test_me_cmp_quant_metrics_batch(sim, refo, orc):
    """quant_psnr / bit / rd (libav_b200/csrc/me_cmp_enc.cu, host-compiled): the batched call against the compiled reference's me_cmp.c"""
    import numpy as np
    import enc_cases
    _enc_protos(sim)

    def run_batch(kind, sidx, handle, cur, ref, recs, h):      # host simulation: "device memory" is host memory
        out, last = np.zeros(len(recs), np.int32), np.zeros(len(recs), np.int32)
        assert sim.ff_me_cmp_enc_batch_cuda(kind, sidx, handle, cur.ctypes.data, ref.ctypes.data, cur.strides[0], h, recs.ctypes.data, len(recs),
                                            out.ctypes.data, last.ctypes.data, None) == 0
        return out, last
    assert enc_cases.batch_cases(sim, run_batch, refo, orc, n=16) > 6000
    assert sim.ff_me_cmp_enc_batch_cuda(13, 0, None, None, None, 0, 8, None, 0, None, None, None) == -1
    sim.avb200_clear_error()


def test_me_cmp_quant_metrics_slots(sim, refo, orc):
    """ff_me_cmp_enc_init_cuda: MECmpContext.quant_psnr / bit / rd over a live (changing) encoder state, host-compiled"""
    import enc_cases
    _enc_protos(sim)
    assert enc_cases.slot_cases(sim, refo, orc) > 800
    sim.avb200_clear_error()


def test_me_cmp_enc_tables_at_a_reused_address(sim, refo, orc):
    """the VLC length tables are found by host address: other tables announced at an address that held some before (here rewritten in place) must be
    taken anew -- by ff_me_cmp_enc_init_cuda and by ff_me_cmp_enc_state_cuda (host-compiled; tests/test_zz_gpu_late_slots.py has the GPU twin)"""
    import enc_cases as E
    from libav_b200 import tables
    _enc_protos(sim)
    T = E.Tables(4)
    u8p = C.POINTER(C.c_uint8)
    for round_ in range(2):
        if round_:
            T2 = E.Tables(99)
            for name in ("intra_len", "intra_last", "inter_len", "inter_last", "luma_dc"):
                getattr(T, name)[:] = getattr(T2, name)
        enc = E.FakeEncoder(T)
        table = tables.MECmpContext()
        key = C.c_void_p(enc.key.ctypes.data)
        label, st = E.states(T)[5]
        enc.load(st, refo)
        assert sim.ff_me_cmp_enc_init_cuda(C.byref(table), key, C.byref(enc.view)) == 0
        cur, rf = E.block_pairs(6, seed=35)
        want, wside = E.oracle_scores(refo, 15, 1, st, cur, rf, 6, 8, h263_guard=orc)
        n = 0
        for i in range(6):
            if want[i] is None:
                continue
            enc.ints[6], enc.ints[8] = st.mb_intra, -2
            a = C.cast(cur.ctypes.data + 16 * i * cur.strides[0] + 8, u8p)
            b = C.cast(rf.ctypes.data + 16 * i * rf.strides[0] + 8, u8p)
            assert table.bit[1](key, a, b, cur.strides[0], 8) == want[i], (round_, i)
            n += 1
        assert n >= 3
        sim.ff_me_cmp_enc_uninit_cuda(key)
        p, _, _, _ = E.product_state(st, refo)
        vlc = E.vlc_tables(T)
        handle = sim.ff_me_cmp_enc_state_cuda(C.byref(p), C.byref(vlc))
        assert handle
        recs = np.array([[16 * i * cur.strides[0] + 8, 16 * i * rf.strides[0] + 8] for i in range(6)], np.uint32)
        got, last = np.zeros(6, np.int32), np.zeros(6, np.int32)
        assert sim.ff_me_cmp_enc_batch_cuda(15, 1, handle, cur.ctypes.data, rf.ctypes.data, cur.strides[0], 8, recs.ctypes.data, 6, got.ctypes.data, last.ctypes.data, None) == 0
        for i in range(6):
            assert want[i] is None or int(got[i]) == want[i], (round_, "batch", i)
        sim.ff_me_cmp_enc_state_free_cuda(handle)


@pytest.mark.parametrize("bits", [8, 9, 10])
def test_h264_pred_422(sim, refo, bits):
    """chroma_format_idc 2: the 8 x 16 entries of pred8x8[] / pred8x8_add[] (libav_b200/csrc/h264pred_hbd.cu, host-compiled), 8 / 9 / 10 bit"""
    import hbd_cases
    assert hbd_cases.pred422_compare(hbd_cases.Pred422Callee(sim.hostsim_h264_pred_install_422), refo, bits, seed=2) > 150
    assert sim.avb200_last_error().decode() == ""


@pytest.mark.parametrize("bits,c422", [(9, 0), (9, 1), (10, 0), (10, 1), (8, 1)])
def test_h264_hbd_batch_residual_and_mc(sim, refo, bits, c422):
    """ff_h264_idct_add_mb_batch_hbd_cuda / ff_h264_mc_batch_hbd_cuda (libav_b200/csrc/h264_hbd_batch.cu, host-compiled) on 9 / 10-bit pictures,
    4:2:0 and 4:2:2, against the compiled reference's BIT_DEPTH > 8 functions applied in the reference's order"""
    import numpy as np
    import h264_hbd_util as hh
    from libav_b200 import synth
    sim.ff_h264_idct_add_mb_batch_hbd_cuda.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t] + [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_void_p]
    sim.ff_h264_mc_batch_hbd_cuda.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_size_t] + [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_void_p]
    for mb_w, mb_h in ((3, 2), (7, 5)):
        y, cb, cr = hh.picture(mb_w, mb_h, bits, c422, seed=5)
        rec, coeffs, nnzc = hh.residual_work(mb_w, mb_h, bits, c422, y, cb, seed=mb_w + bits)
        wy, wcb, wcr, wco = y.copy(), cb.copy(), cr.copy(), coeffs.copy()
        hh.oracle_residual(refo, bits, c422, rec, wco, nnzc, wy, wcb, wcr)
        assert sim.ff_h264_idct_add_mb_batch_hbd_cuda(bits, 1 + c422, rec.ctypes.data, len(rec), coeffs.ctypes.data, 768, nnzc.ctypes.data, y.ctypes.data,
                                                      cb.ctypes.data, cr.ctypes.data, y.strides[0], cb.strides[0], None) == 0
        assert np.array_equal(y, wy) and np.array_equal(cb, wcb) and np.array_equal(cr, wcr) and np.array_equal(coeffs, wco)
        refs = [hh.picture(mb_w, mb_h, bits, c422, seed=11), hh.picture(mb_w, mb_h, bits, c422, seed=12)]
        mrec = synth.h264_mc_work(mb_w, mb_h, seed=mb_h + bits, max_mv=64 if mb_w > 4 else 24, avg_second=True)
        y, cb, cr = hh.picture(mb_w, mb_h, bits, c422, seed=13)
        wy, wcb, wcr = y.copy(), cb.copy(), cr.copy()
        hh.oracle_mc(refo, bits, c422, mrec, refs, wy, wcb, wcr)
        planes = np.array([[p.ctypes.data for p in r] for r in refs], dtype=np.uint64)
        assert sim.ff_h264_mc_batch_hbd_cuda(bits, 1 + c422, mrec.ctypes.data, len(mrec), planes.ctypes.data, y.ctypes.data, cb.ctypes.data, cr.ctypes.data,
                                             y.strides[0], cb.strides[0], 16 * mb_w, 16 * mb_h, None) == 0
        assert np.array_equal(y, wy), "luma"
        assert np.array_equal(cb, wcb) and np.array_equal(cr, wcr), "chroma"
    assert sim.avb200_last_error().decode() == ""


@pytest.mark.parametrize("bits", [9, 10])
def test_h264_hbd_batch_weight_and_dc(sim, refo, bits):
    """ff_h264_weight_batch_hbd_cuda / ff_h264_dc_dequant_batch_hbd_cuda (host-compiled) against the compiled reference's BIT_DEPTH > 8 functions"""
    import h264_hbd_util as hh
    sim.ff_h264_weight_batch_hbd_cuda.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    sim.ff_h264_dc_dequant_batch_hbd_cuda.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]

    def run_weight(b, rec, plane, src):
        assert sim.ff_h264_weight_batch_hbd_cuda(b, rec.ctypes.data, len(rec), plane.ctypes.data, src.ctypes.data if src is not None else None, plane.strides[0], None) == 0
        return plane

    def run_dc(c422, recs, coeffs, luma_dc):
        assert sim.ff_h264_dc_dequant_batch_hbd_cuda(1 + c422, recs.ctypes.data, len(recs), coeffs.ctypes.data, 768, luma_dc.ctypes.data, None) == 0
        return coeffs
    hh.weight_dc_cases(run_weight, run_dc, refo, bits)
    assert sim.avb200_last_error().decode() == ""
