"""CPU: the loop-filter slots of the product's H264DSPContext (host simulation of libav_b200/csrc/slots.cu) under the reference's own
deblocking driver -- see tests/h264_dropin_cases.py."""
import pytest

from test_hostsim_slots_cpu import sim          # noqa: F401


def test_loop_filter_slots_under_the_reference_driver(sim, refo):
    import h264_dropin_cases as D
    assert D.check(refo, sim) == 18
    assert sim.avb200_last_error().decode() == ""


@pytest.mark.parametrize("bits", [9, 10])
def test_loop_filter_slots_under_the_reference_driver_hbd(sim, refo, bits):
    """the 9 / 10-bit slots (libav_b200/csrc/slots_hbd.cu) on uint16 planes, the driver deciding with qp_bd_offset on QP'-scale side information"""
    import h264_dropin_cases as D
    if not refo.has("h264_deblock_picture_with_hbd"):
        pytest.skip("oracle/_ref was built before h264_deblock_picture_with_hbd existed")
    assert D.check(refo, sim, bits=bits) == 18
    assert sim.avb200_last_error().decode() == ""
