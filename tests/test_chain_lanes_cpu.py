"""The lane entry points of both chain engines (dspi_chain(q)_lane_*) and their Python wrappers, without a GPU: every entry
point refuses a NULL handle before it looks at any other argument, and both engine classes carry the wrappers."""
import ctypes as C
import os
import re

import pytest

from dspi_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
METHODS = ["lane_open", "lane_close", "lane_process_packets_device", "lane_process_subframes_device", "lane_stream", "lane_sync"]


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(api.LIB_PATH):
        from dspi_b200.build import build
        build()
    return api.lib()


@pytest.mark.parametrize("pre", ["dspi_chain", "dspi_chainq"])
def test_lane_entry_points_reject_a_null_handle(lib, pre):
    fn = lambda name: getattr(lib, pre + "_" + name)
    buf = (C.c_uint8 * 4096)()
    table = (C.c_uint16 * 1)(48)
    lane = C.c_uint32(7)
    for inst0, n in ((0, 64), (32, 1), (0, 0), (0xFFFFFFC0, 128)):   # the handle is refused before the window is looked at
        assert fn("lane_open")(None, inst0, n, C.byref(lane)) == -22
        assert b"null argument" in lib.dspi_last_error()
        assert fn("lane_open")(None, inst0, n, None) == -22
    assert lane.value == 7                                               # nothing written
    for form in ("packets", "subframes"):
        f = fn("lane_process_%s_device" % form)
        for ln, inst0, n in ((0, 0, 1), (15, 64, 17), (16, 32, 1), (0xFFFFFFFF, 0, 0)):
            assert f(None, ln, inst0, n, buf, 24, 1, table, buf, buf, buf) == -22
            assert b"null argument" in lib.dspi_last_error()
            assert f(None, ln, inst0, n, None, 24, 1, None, None, None, None) == -22
    for ln in (0, 15, 16, 0xFFFFFFFF):
        assert fn("lane_close")(None, ln) == -22
        assert b"null argument" in lib.dspi_last_error()
        assert fn("lane_sync")(None, ln) == -22
        assert fn("lane_stream")(None, ln) is None


def test_header_sets_the_lane_limit():
    hdr = open(os.path.join(ROOT, "include", "dspi_b200.h")).read()
    assert re.search(r"#define\s+DSPI_CHAIN_MAX_LANES\s+16\b", hdr)


@pytest.mark.parametrize("cls", [api.ChainEngine, api.ChainEngineQ28])
def test_both_engine_classes_have_the_lane_wrappers(cls):
    for m in METHODS:
        assert callable(getattr(cls, m, None)), m
