"""Deblocking DECISIONS of 9 / 10-bit pictures: the plain-C port (oracle/port/orc_h264lf.c) against the reference's own h264_loopfilter.c
(oracle/_ref, recording slots) with sps->bit_depth_luma set, on side information in the decoder's QP' scale (synth.h264_deblock_info with
bit_depth): qscale 0 (I_PCM) to 51 + qp_bd_offset, qp_thresh with its bit-depth term, chroma_qp_index_offset and alpha / beta offsets
out to +-12.  The 8-bit cases live in test_oracle_h264lf_cpu.py; these reuse its case lists."""
import numpy as np
import pytest

from libav_b200 import synth
from oracle.loader import ptr
from test_oracle_h264lf_cpu import C422_CASES, CASES, FIELD_CASES, as_field, run as run8

ids = lambda c: "-".join("%s%s" % kv for kv in c.items())


def run(o, d, bit_depth=None):
    """h264_deblock_params_hbd: the decisions for side information d at bit_depth (default: the depth d was drawn for)"""
    out = np.zeros((d["mb_w"] * d["mb_h"], 104), np.uint8)
    rc = o.h264_deblock_params_hbd(bit_depth or d["bit_depth"], d["mb_w"], d["mb_h"], ptr(d["mb_type"]), ptr(d["qscale"]), ptr(d["nnz"]),
                                   ptr(d["cbp"]), ptr(d["slice_table"]), ptr(d["mv0"]), ptr(d["mv1"]), ptr(d["ref0"]), ptr(d["ref1"]),
                                   ptr(d["slice_params"]), d["n_slices"], ptr(d["chroma_qp_table"]), d["cabac"], d["t8x8"], ptr(out))
    assert rc == 0
    return out


def run422(o, d):
    """chroma_format_idc 2 at d's bit depth: (104-byte records, 52-byte records of the four horizontal chroma edges)"""
    ext = np.full((d["mb_w"] * d["mb_h"], 52), 0xEE, np.uint8)
    try:
        o.h264_deblock_chroma422(ptr(ext))
        rec = run(o, d)
    finally:
        o.h264_deblock_chroma422(None)
    return rec, ext


def hbd_oracle(o):
    """o when it decides at 9 / 10 bit, else the port (an oracle/_ref built from sources older than h264_deblock_params_hbd lacks it)"""
    from oracle import loader
    return o if o.has("h264_deblock_params_hbd") else loader.port()


@pytest.fixture
def refo_hbd(refo):
    if not refo.has("h264_deblock_params_hbd"):
        pytest.skip("oracle/_ref was built before h264_deblock_params_hbd existed")
    return refo


def _same(a, b, what):
    bad = np.argwhere((a != b).any(axis=1))
    assert not len(bad), (what, bad[:4].ravel().tolist(), a[bad[0, 0]].tolist(), b[bad[0, 0]].tolist())


@pytest.mark.parametrize("case", CASES, ids=ids)
@pytest.mark.parametrize("bits", [9, 10])
def test_port_matches_reference_decisions_hbd(orc, refo_hbd, bits, case):
    for (mw, mh) in ((11, 9), (1, 1), (2, 5), (20, 3)):
        d = synth.h264_deblock_info(mw, mh, bit_depth=bits, **case)
        _same(run(refo_hbd, d), run(orc, d), (mw, mh))


@pytest.mark.parametrize("case", FIELD_CASES, ids=ids)
@pytest.mark.parametrize("bits", [9, 10])
def test_field_pictures_hbd(orc, refo_hbd, bits, case):
    for (mw, mh) in ((11, 9), (2, 5), (20, 3)):
        d = as_field(synth.h264_deblock_info(mw, mh, bit_depth=bits, **case))
        try:
            refo_hbd.h264_deblock_picture_structure(1); orc.h264_deblock_picture_structure(1)
            a, b = run(refo_hbd, d), run(orc, d)
        finally:
            refo_hbd.h264_deblock_picture_structure(0); orc.h264_deblock_picture_structure(0)
        _same(a, b, (mw, mh))


@pytest.mark.parametrize("case", C422_CASES, ids=ids)
@pytest.mark.parametrize("bits", [9, 10])
def test_chroma422_hbd(orc, refo_hbd, bits, case):
    for (mw, mh) in ((11, 9), (2, 5), (20, 3)):
        d = synth.h264_deblock_info(mw, mh, bit_depth=bits, **case)
        (a, ea), (b, eb) = run422(refo_hbd, d), run422(orc, d)
        _same(a, b, (mw, mh))
        _same(ea, eb, ("ext", mw, mh))


def _oracles(orc):
    """the port, and the compiled reference when it has the _hbd calls"""
    from oracle import loader
    r = loader.ref()
    return [orc] + ([r] if r is not None and r.has("h264_deblock_params_hbd") else [])


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_8_bit_equals_the_8_bit_call(orc, case):
    """h264_deblock_params_hbd at bit_depth 8 writes what h264_deblock_params writes, in the port and in the reference"""
    for (mw, mh) in ((11, 9), (1, 1)):
        d = synth.h264_deblock_info(mw, mh, **case)
        for o in _oracles(orc):
            assert np.array_equal(run(o, d, bit_depth=8), run8(o, d)), (o.prefix, mw, mh)


def test_bit_depth_is_refused_outside_8_to_10(orc):
    d = synth.h264_deblock_info(2, 2)
    for o in _oracles(orc):
        for bits in (7, 11, 12):
            out = np.full((4, 104), 0xAB, np.uint8)
            assert o.h264_deblock_params_hbd(bits, 2, 2, ptr(d["mb_type"]), ptr(d["qscale"]), ptr(d["nnz"]), ptr(d["cbp"]), ptr(d["slice_table"]),
                                             ptr(d["mv0"]), ptr(d["mv1"]), ptr(d["ref0"]), ptr(d["ref1"]), ptr(d["slice_params"]), d["n_slices"],
                                             ptr(d["chroma_qp_table"]), d["cabac"], d["t8x8"], ptr(out)) == -1
            assert (out == 0xAB).all()


def _offset_of(bits, row):
    """the chroma_qp_index_offset a chroma_qp_table row was built with"""
    hits = [o for o in range(-12, 13) if np.array_equal(synth.h264_chroma_qp_table(bits, o), row)]
    assert len(hits) == 1
    return hits[0]


@pytest.mark.parametrize("bits", [9, 10])
def test_side_information_in_the_decoders_scale(bits):
    """what the 9 / 10-bit side information must contain for the decisions tests to mean anything"""
    bd = 6 * (bits - 8)
    max_qp = 51 + bd
    qs, near, offs, pcm = [], [], [], 0
    for seed in range(1, 9):
        d = synth.h264_deblock_info(11, 9, seed=seed, n_slices=4, bit_depth=bits)
        real = d["slice_table"] != 0xFFFF
        q = d["qscale"][real].astype(int)
        qs.append(q)
        pcm += int((d["mb_type"] == synth.MB_INTRA_PCM).sum())
        assert (d["qscale"][d["mb_type"] == synth.MB_INTRA_PCM] == 0).all()
        sp = d["slice_params"]
        offs += sp[:, :2].ravel().tolist()
        cb, cr = (_offset_of(bits, d["chroma_qp_table"][t]) for t in (0, 1))
        assert cb != cr
        assert (sp[:, 4] == 15 - np.minimum(sp[:, 0], sp[:, 1]) - max(0, cb, cr) + bd).all()          # h264_slice.c:1815-1820
        near.append(np.abs(q - sp[d["slice_table"][real], 4]) <= 2)
    q = np.concatenate(qs)
    assert q.min() == 0 and q.max() == max_qp and (q > 51).mean() > 0.1
    assert np.concatenate(near).mean() > 0.2
    assert pcm and min(offs) == -12 and max(offs) == 12


def test_chroma_qp_table_in_the_decoders_scale():
    """QP'c = QPc(Clip3(-QpBdOffsetC, 51, QP'y - QpBdOffsetY + offset)) + QpBdOffsetC at a few points worked out by hand"""
    assert np.array_equal(synth.h264_chroma_qp_table(8, 0)[:52], synth.H264_CHROMA_QP)
    t10 = synth.h264_chroma_qp_table(10, 0)
    assert t10[:42].tolist() == list(range(42)) and t10[42] == 41 and t10[63] == 51
    t9 = synth.h264_chroma_qp_table(9, -12)
    assert t9[:18].tolist() == [0] * 13 + [1, 2, 3, 4, 5] and t9[57] == 35 + 6 and not t9[58:].any()     # qPI 39 -> QPc 35


@pytest.mark.parametrize("bits", [9, 10])
def test_the_8_bit_model_is_wrong_on_high_bit_depth_data(orc, bits):
    """teeth: on side information in the QP' scale, decisions taken as if it were 8-bit (the table index without - qp_bd_offset) differ from
    the decisions at the stream's depth in most records that filter anything"""
    filtered = differ = 0
    for seed in range(1, 5):
        d = synth.h264_deblock_info(20, 12, seed=seed, bipred=bool(seed & 1), bit_depth=bits)
        a, b = run(orc, d), run(orc, d, bit_depth=8)
        any_edge = (a.view(synth.DEBLOCK_DT)["alpha"].reshape(len(a), -1).any(axis=1) |
                    b.view(synth.DEBLOCK_DT)["alpha"].reshape(len(b), -1).any(axis=1))
        filtered += int(any_edge.sum())
        differ += int(((a != b).any(axis=1) & any_edge).sum())
    assert filtered > 500 and differ > 0.5 * filtered, (differ, filtered)
