"""dspi_chain(q)_copy_instances refuses a NULL engine and NULL lists before any device work (runs without a GPU)."""
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
def test_null_engine_and_null_lists_are_refused(lib, pre):
    fn = getattr(lib, pre + "_copy_instances")
    src = (C.c_uint32 * 3)(0, 1, 2)
    dst = (C.c_uint32 * 3)(5, 6, 7)
    assert fn(None, 3, src, dst) == -22
    assert b"null argument" in lib.dspi_last_error()
    assert fn(None, 3, None, dst) == -22
    assert fn(None, 3, src, None) == -22
    assert fn(None, 0, None, None) == -22
    assert list(src) == [0, 1, 2] and list(dst) == [5, 6, 7]
