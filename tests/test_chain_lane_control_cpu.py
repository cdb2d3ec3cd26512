"""The lane control calls of both chain engines (dspi_chain(q)_lane_edit_bulk_device, _lane_set_preset_mute,
_lane_set_spdif_tx, _lane_reset_instances) and their Python wrappers, without a GPU: every entry point refuses a NULL
handle before it looks at any other argument and writes nothing, and both engine classes carry the wrappers."""
import ctypes as C
import os

import numpy as np
import pytest

from dspi_b200 import api, layouts as L

METHODS = ["lane_edit_bulk_device", "lane_set_preset_mute", "lane_set_spdif_tx", "lane_reset_instances"]


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(api.LIB_PATH):
        from dspi_b200.build import build
        build()
    return api.lib()


@pytest.mark.parametrize("pre", ["dspi_chain", "dspi_chainq"])
def test_lane_control_entry_points_reject_a_null_handle(lib, pre):
    fn = lambda name: getattr(lib, pre + "_" + name)                    # noqa: E731
    edits = np.concatenate([L.bulk_edit(3, ("outputs", 0, "gain_db"), np.float32(-6.0))] * 2)
    res = np.full(2, 7, np.int32)
    states = np.zeros(4, L.PRESET_MUTE)
    states["smooth_gain"] = 0.5
    tx = np.zeros(4, L.SPDIF_TX)
    tx["block_pos"] = 3
    ed, st, tp, rp = (x.ctypes.data_as(C.c_void_p) for x in (edits, states, tx, res))
    before = (edits.tobytes(), states.tobytes(), tx.tobytes())
    for ln, inst0, n in ((0, 0, 1), (15, 64, 4), (16, 32, 1), (0xFFFFFFFF, 0xFFFFFFF0, 0x20)):   # refused before lane and window
        for args in ((ed, 0, C.c_float(48000.0), rp), (None, 1, C.c_float(-1.0), None)):
            assert fn("lane_edit_bulk_device")(None, ln, 2, args[0], args[1], args[2], args[3]) == -22
            assert b"null argument" in lib.dspi_last_error()
        for p in (st, None):
            assert fn("lane_set_preset_mute")(None, ln, inst0, n, p, 48000) == -22
            assert b"null argument" in lib.dspi_last_error()
        for p in (tp, None):
            assert fn("lane_set_spdif_tx")(None, ln, inst0, n, p) == -22
            assert b"null argument" in lib.dspi_last_error()
        assert fn("lane_reset_instances")(None, ln, inst0, n) == -22
        assert b"null argument" in lib.dspi_last_error()
    assert res.tolist() == [7, 7]                                        # nothing written
    assert (edits.tobytes(), states.tobytes(), tx.tobytes()) == before


@pytest.mark.parametrize("cls", [api.ChainEngine, api.ChainEngineQ28])
def test_both_engine_classes_have_the_lane_control_wrappers(cls):
    for m in METHODS:
        assert callable(getattr(cls, m, None)), m
