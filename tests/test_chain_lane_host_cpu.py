"""The lane host calls of both chain engines (dspi_chain(q)_lane_process_packets_host, _lane_process_subframes_host) and
their Python wrapper, without a GPU: every entry point refuses a NULL handle before it looks at any other argument and
writes nothing, and both engine classes carry the wrapper."""
import ctypes as C
import os

import numpy as np
import pytest

from dspi_b200 import api


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(api.LIB_PATH):
        from dspi_b200.build import build
        build()
    return api.lib()


@pytest.mark.parametrize("pre", ["dspi_chain", "dspi_chainq"])
@pytest.mark.parametrize("form", ["packets", "subframes"])
def test_lane_host_entry_points_reject_a_null_handle(lib, pre, form):
    fn = getattr(lib, "%s_lane_process_%s_host" % (pre, form))
    pcm = np.full(4096, 0x3C, np.uint8)                                # pageable: refused later, if ever
    out = np.full(1 << 16, 0xA5, np.uint8)
    table = np.array([48, 48], np.uint16)
    p, o, t = (x.ctypes.data_as(C.c_void_p) for x in (pcm, out, table))
    for ln, inst0, n, bd, nk in ((0, 0, 1, 24, 2), (15, 64, 2, 16, 1), (16, 32, 3, 20, 0), (0xFFFFFFFF, 0xFFFFFFC0, 0x80, 24, 2)):
        for args in ((p, bd, nk, t, o, o, o), (None, bd, nk, None, None, None, None)):
            assert fn(None, ln, inst0, n, *args) == -22
            assert b"null argument" in lib.dspi_last_error()
    assert (pcm == 0x3C).all() and (out == 0xA5).all()                 # nothing written
    assert table.tolist() == [48, 48]


@pytest.mark.parametrize("cls", [api.ChainEngine, api.ChainEngineQ28])
def test_both_engine_classes_have_the_lane_host_wrapper(cls):
    assert callable(getattr(cls, "lane_process_packets_host", None))


def test_the_wrapper_takes_pinned_buffers_only():
    with pytest.raises(TypeError):
        api._pinned(np.zeros((2, 8), np.uint8))
