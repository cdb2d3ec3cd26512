"""The lane configuration calls of both chain engines (dspi_chain(q)_lane_apply_bulk_device, _lane_apply_preset_device,
_lane_set_rate_device) and their Python wrappers, without a GPU: every entry point refuses a NULL handle before it looks
at any other argument and writes nothing, and both engine classes carry the wrappers."""
import ctypes as C
import os

import numpy as np
import pytest

from dspi_b200 import api, layouts as L

METHODS = ["lane_apply_bulk_device", "lane_apply_preset_device", "lane_set_rate_device"]


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(api.LIB_PATH):
        from dspi_b200.build import build
        build()
    return api.lib()


@pytest.mark.parametrize("pre", ["dspi_chain", "dspi_chainq"])
def test_lane_config_entry_points_reject_a_null_handle(lib, pre):
    fn = lambda name: getattr(lib, pre + "_" + name)                    # noqa: E731
    packets = np.zeros(2, L.WIRE_BULK)
    host = np.zeros(2, L.BULK_HOST)
    images = np.full((2, 4096), 0xA5, np.uint8)
    load = np.zeros(2, L.PRESET_LOAD)
    rates = np.array([48000.0, float("nan")], np.float32)
    res = np.full(2, 7, np.int32)
    pk, hp, ip, lp, rt, rp = (x.ctypes.data_as(C.c_void_p) for x in (packets, host, images, load, rates, res))
    before = (packets.tobytes(), host.tobytes(), images.tobytes(), load.tobytes(), rates.tobytes())
    for ln, inst0, n in ((0, 0, 1), (15, 64, 2), (16, 32, 1), (0xFFFFFFFF, 0xFFFFFFF0, 0x20)):   # refused before lane and window
        for p, h, rate, r in ((pk, hp, C.c_float(48000.0), rp), (None, None, C.c_float(-1.0), None)):
            assert fn("lane_apply_bulk_device")(None, ln, inst0, n, p, h, 0, rate, r) == -22
            assert b"null argument" in lib.dspi_last_error()
        for i, stride, ld, h, rate, r in ((ip, 4096, lp, hp, C.c_float(48000.0), rp), (None, 0, None, None, C.c_float(0.0), None)):
            assert fn("lane_apply_preset_device")(None, ln, inst0, n, i, C.c_size_t(stride), ld, h, rate, r) == -22
            assert b"null argument" in lib.dspi_last_error()
        for r, out in ((rt, rp), (None, None)):
            assert fn("lane_set_rate_device")(None, ln, inst0, n, r, out) == -22
            assert b"null argument" in lib.dspi_last_error()
    assert res.tolist() == [7, 7]                                        # nothing written
    assert (packets.tobytes(), host.tobytes(), images.tobytes(), load.tobytes(), rates.tobytes()) == before


@pytest.mark.parametrize("cls", [api.ChainEngine, api.ChainEngineQ28])
def test_both_engine_classes_have_the_lane_config_wrappers(cls):
    for m in METHODS:
        assert callable(getattr(cls, m, None)), m
