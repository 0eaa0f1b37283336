"""CPU: the per-line SwsContext slots of the product (host simulation of libav_b200/csrc/sws_slots.cu) plugged into a real reference
SwsContext and driven by the reference's unmodified swscale() -- see tests/sws_dropin_cases.py."""
import ctypes as C

import numpy as np
import pytest

from test_hostsim_slots_cpu import sim          # noqa: F401  (the fixture that builds / loads tests/hostsim/libhostsim.so)


def test_slots_under_the_reference_scheduler(sim, refo):
    import sws_dropin_cases as D

    def make_ctx(sf, w, h, df, dw, dh, flags):
        ctx = sim.sws_getContext_cuda(w, h, sf, dw, dh, df, flags, None, None, None)
        assert ctx, (sf, df, hex(flags), sim.avb200_last_error())
        return ctx
    assert D.check(refo, sim, make_ctx, sim.sws_freeContext_cuda) == 84
    assert sim.avb200_last_error().decode() == ""


def test_high_bit_depth_sources_keep_the_c_slots(sim, refo):
    """a 9 / 10 / 16-bit planar source: the reference installs hScale16To15_c and per-line dither rows the hook cannot see -- it must
    refuse (return -1, every slot NULL, a message) instead of installing the 8-bit line functions"""
    from libav_b200 import tables
    for sf in (62, 64, 47):                                    # yuv420p9le, yuv420p10le, yuv420p16le
        for df in (0, 2):                                      # yuv420p, rgb24
            cuda = sim.sws_getContext_cuda(64, 48, sf, 96, 64, df, 4, None, None, None)
            assert cuda, sim.avb200_last_error()
            c = refo.sws_open(sf, 64, 48, df, 96, 64, 4)
            assert c
            t = tables.SwsLineSlotsCUDA()
            assert sim.ff_sws_init_swscale_cuda(C.c_void_p(c), C.c_void_p(cuda), C.byref(t)) == -1
            assert b"high-bit-depth" in sim.avb200_last_error()
            assert all(not C.cast(getattr(t, name), C.c_void_p).value for name, _ in tables.SwsLineSlotsCUDA._fields_)
            sim.avb200_clear_error()
            refo.sws_close(c)
            sim.sws_freeContext_cuda(cuda)
