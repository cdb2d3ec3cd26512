"""Both chain engines refuse a NULL handle on every entry point that takes one, before any device work (runs without a
GPU).  The two engines share one host implementation (dspi_b200/csrc/chain_host.cuh), so each prefix is checked on its
own: the forwards are written out per engine.  The response calls are covered by test_response_cpu.py."""
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
def test_every_handle_taking_entry_point_rejects_null(lib, pre):
    fn = lambda name: getattr(lib, pre + "_" + name)
    buf = (C.c_uint8 * 4096)()                                  # every other pointer argument valid: the handle is what is refused
    fs, size = C.c_float(48000.0), C.c_size_t(len(buf))
    calls = {
        "reset_state": (), "sync": (), "sm_partition": (buf, buf),
        "set_params": (0, 1, buf), "set_dynamics_device": (0, 1, buf, fs), "set_preset_mute": (0, 1, buf, 48000), "get_preset_mute": (0, 1, buf),
        "upload_biquads": (0, 1, buf), "download_biquads": (0, 1, buf), "set_eq_params_device": (0, 1, buf, fs),
        "apply_bulk_device": (0, 1, buf, buf, 0, fs, buf), "collect_bulk_device": (0, 1, buf, buf, buf),
        "apply_preset_device": (0, 1, buf, size, buf, buf, fs, buf), "collect_preset_device": (0, 1, buf, buf, size, buf),
        "set_spdif_tx": (0, 1, buf), "get_spdif_tx": (0, 1, buf),
        "process_host": (buf, 16, 1, 1, buf, buf, buf), "process_device": (buf, 16, 1, 1, buf, buf, buf),
        "process_packets_host": (buf, 16, 1, buf, buf, buf, buf), "process_packets_device": (buf, 16, 1, buf, buf, buf, buf),
        "process_subframes_host": (buf, 16, 1, buf, buf, buf, buf), "process_subframes_device": (buf, 16, 1, buf, buf, buf, buf),
        "state_export": (buf, size), "state_import": (buf, size),
    }
    for name, args in calls.items():
        assert fn(name)(None, *args) == -22, name
        assert b"null argument" in lib.dspi_last_error(), name
    assert fn("destroy")(None) == 0
    assert fn("state_size")(None) == 0
    assert fn("stream")(None) is None
    assert fn("launch_count")(None) == 0
