"""The per-instance lifecycle entry points of both chain engines (_instance_image_size, _export_instances,
_import_instances, _reset_instances) refuse a NULL handle before any device work, as every other handle-taking entry point
does (test_chain_null_handle_cpu.py).  Runs without a GPU."""
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
def test_instance_lifecycle_entry_points_reject_null(lib, pre):
    fn = lambda name: getattr(lib, pre + "_" + name)                  # noqa: E731
    buf = (C.c_uint8 * 4096)()
    size = C.c_size_t(len(buf))
    calls = {"export_instances": (0, 1, buf, size), "import_instances": (0, 1, buf, size), "reset_instances": (0, 1)}
    for name, args in calls.items():
        assert fn(name)(None, *args) == -22, name
        assert b"null argument" in lib.dspi_last_error(), name
        assert fn(name)(None, 0, 0, *args[2:]) == -22, name            # before the n == 0 shortcut
    assert fn("instance_image_size")(None) == 0
