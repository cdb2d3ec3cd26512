"""The eight instance-range process entry points (dspi_chain(q)_process_packets_range_* / _process_subframes_range_*) and
their Python wrappers, without a GPU: every entry point is exported, refuses a NULL handle or a NULL pcm before any device
work, and both engine classes carry the four wrappers."""
import ctypes as C

import pytest

from dspi_b200 import api

FORMS = ["process_packets_range_host", "process_packets_range_device", "process_subframes_range_host", "process_subframes_range_device"]


@pytest.fixture(scope="module")
def lib():
    import os
    if not os.path.exists(api.LIB_PATH):
        from dspi_b200.build import build
        build()
    return api.lib()


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("pre", ["dspi_chain", "dspi_chainq"])
def test_range_entry_points_reject_null_handle_and_pcm(lib, pre, form):
    fn = getattr(lib, pre + "_" + form)
    buf = (C.c_uint8 * 4096)()
    table = (C.c_uint16 * 1)(48)
    for inst0, n in ((0, 1), (64, 17), (32, 1), (0, 0)):       # the handle is refused before the window is looked at
        assert fn(None, inst0, n, buf, 24, 1, table, buf, buf, buf) == -22
        assert b"null argument" in lib.dspi_last_error()
        assert fn(None, inst0, n, None, 24, 1, table, buf, buf, buf) == -22


@pytest.mark.parametrize("cls", [api.ChainEngine, api.ChainEngineQ28])
def test_both_engine_classes_have_the_range_wrappers(cls):
    for form in FORMS:
        assert callable(getattr(cls, form, None)), form
