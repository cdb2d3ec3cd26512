"""The lane read calls of both chain engines (dspi_chain(q)_lane_collect_bulk_device, _lane_collect_preset_device,
_lane_export_instances, _lane_response_device, _lane_get_preset_mute, _lane_get_spdif_tx) and their Python wrappers,
without a GPU: every entry point refuses a NULL handle before it looks at any other argument and writes nothing, and both
engine classes carry the wrappers."""
import ctypes as C
import os

import numpy as np
import pytest

from dspi_b200 import api

METHODS = ["lane_collect_bulk_device", "lane_collect_preset_device", "lane_export_instances", "lane_response_device",
           "lane_get_preset_mute", "lane_get_spdif_tx"]


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(api.LIB_PATH):
        from dspi_b200.build import build
        build()
    return api.lib()


@pytest.mark.parametrize("pre", ["dspi_chain", "dspi_chainq"])
def test_lane_read_entry_points_reject_a_null_handle(lib, pre):
    fn = lambda name: getattr(lib, pre + "_" + name)                    # noqa: E731
    out = np.full(1 << 16, 0xA5, np.uint8)                              # stands for every output
    slots = np.array([1, 2], np.uint8)
    freqs = np.array([100.0, float("nan")], np.float32)
    op, sp, fp = (x.ctypes.data_as(C.c_void_p) for x in (out, slots, freqs))
    for ln, inst0, n in ((0, 0, 1), (15, 64, 2), (16, 32, 1), (0xFFFFFFFF, 0xFFFFFFF0, 0x20)):   # refused before lane and window
        for o, s, f, stride, fs in ((op, sp, fp, 4096, C.c_float(48000.0)), (None, None, None, 0, C.c_float(-1.0))):
            calls = [fn("lane_collect_bulk_device")(None, ln, inst0, n, o, o, o),
                     fn("lane_collect_preset_device")(None, ln, inst0, n, s, o, C.c_size_t(stride), o),
                     fn("lane_export_instances")(None, ln, inst0, n, o, C.c_size_t(stride)),
                     fn("lane_response_device")(None, ln, inst0, n, f, 2, fs, o),
                     fn("lane_get_preset_mute")(None, ln, inst0, n, o),
                     fn("lane_get_spdif_tx")(None, ln, inst0, n, o)]
            for j, rc in enumerate(calls):
                assert rc == -22, j
            assert b"null argument" in lib.dspi_last_error()
            for name, args in (("lane_response_device", (f, 0, fs, o)), ("lane_export_instances", (o, C.c_size_t(0)))):
                assert fn(name)(None, ln, inst0, n, *args) == -22 and b"null argument" in lib.dspi_last_error(), name
    assert (out == 0xA5).all()                                           # nothing written
    assert slots.tolist() == [1, 2]


@pytest.mark.parametrize("cls", [api.ChainEngine, api.ChainEngineQ28])
def test_both_engine_classes_have_the_lane_read_wrappers(cls):
    for m in METHODS:
        assert callable(getattr(cls, m, None)), m
