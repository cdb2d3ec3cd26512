"""The lane move calls of both chain engines (dspi_chain(q)_lane_import_instances, _lane_copy_instances) and their Python
wrappers, without a GPU: every entry point refuses a NULL handle before it looks at any other argument and writes nothing,
and both engine classes carry the wrappers."""
import ctypes as C
import os

import numpy as np
import pytest

from dspi_b200 import api

METHODS = ["lane_import_instances", "lane_copy_instances"]


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(api.LIB_PATH):
        from dspi_b200.build import build
        build()
    return api.lib()


@pytest.mark.parametrize("pre", ["dspi_chain", "dspi_chainq"])
def test_lane_move_entry_points_reject_a_null_handle(lib, pre):
    fn = lambda name: getattr(lib, pre + "_" + name)                    # noqa: E731
    images = np.full(1 << 16, 0xA5, np.uint8)
    src = np.array([1, 2, 2], np.uint32)
    dst = np.array([3, 3, 1], np.uint32)                                # a duplicate and an overlap: refused later, if ever
    ip, sp, dp = (x.ctypes.data_as(C.c_void_p) for x in (images, src, dst))
    for ln, ln2, inst0, n in ((0, 0, 0, 1), (15, 1, 64, 2), (16, 16, 32, 3), (0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFF0, 0x20)):
        for i, s, d, stride in ((ip, sp, dp, 4096), (None, None, None, 0)):
            assert fn("lane_import_instances")(None, ln, inst0, n, i, C.c_size_t(stride)) == -22
            assert b"null argument" in lib.dspi_last_error()
            assert fn("lane_copy_instances")(None, ln, ln2, n, s, d) == -22
            assert b"null argument" in lib.dspi_last_error()
    assert (images == 0xA5).all()                                       # nothing written
    assert src.tolist() == [1, 2, 2] and dst.tolist() == [3, 3, 1]


@pytest.mark.parametrize("cls", [api.ChainEngine, api.ChainEngineQ28])
def test_both_engine_classes_have_the_lane_move_wrappers(cls):
    for m in METHODS:
        assert callable(getattr(cls, m, None)), m
