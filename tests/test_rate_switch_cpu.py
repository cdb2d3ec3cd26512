"""dspi_chain(q)_set_rate_device refuses a NULL engine and NULL rates before any device work (runs without a GPU)."""
import ctypes as C

import pytest

from dspi_b200 import api


@pytest.fixture(scope="module")
def lib():
    import os
    if not os.path.exists(api.LIB_PATH):
        from dspi_b200.build import build
        build()
    return api.lib()


@pytest.mark.parametrize("pre", ["dspi_chain", "dspi_chainq"])
def test_null_engine_and_null_rates_are_refused(lib, pre):
    fn = getattr(lib, pre + "_set_rate_device")
    rates = (C.c_float * 4)(48000.0, 44100.0, 96000.0, 192000.0)
    results = (C.c_int32 * 4)(77, 77, 77, 77)
    assert fn(None, 0, 4, rates, results) == -22
    assert b"null argument" in lib.dspi_last_error()
    assert fn(None, 0, 4, None, results) == -22
    assert fn(None, 0, 0, None, None) == -22
    assert list(results) == [77] * 4
