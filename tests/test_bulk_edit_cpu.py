"""dspi_chain(q)_edit_bulk_device refuses a NULL engine and NULL edits before any device work; the BULK_EDIT record and the
edit helper of layouts.py follow the C header and WIRE_BULK (runs without a GPU)."""
import ctypes as C

import numpy as np
import pytest

from dspi_b200 import api, layouts as L


@pytest.fixture(scope="module")
def lib():
    import os
    if not os.path.exists(api.LIB_PATH):
        from dspi_b200.build import build
        build()
    return api.lib()


@pytest.mark.parametrize("pre", ["dspi_chain", "dspi_chainq"])
def test_null_engine_and_null_edits_are_refused(lib, pre):
    fn = getattr(lib, pre + "_edit_bulk_device")
    edits = np.concatenate([L.bulk_edit(0, ("outputs", 1, "gain_db"), -3.0), L.bulk_edit(1, ("host", "host_mute"), 1)])
    results = (C.c_int32 * 2)(77, 77)
    ep = edits.ctypes.data_as(C.c_void_p)
    assert fn(None, 2, ep, 0, C.c_float(48000.0), results) == -22
    assert b"null argument" in lib.dspi_last_error()
    assert fn(None, 2, None, 0, C.c_float(48000.0), results) == -22
    assert fn(None, 0, None, 1, C.c_float(48000.0), None) == -22
    assert list(results) == [77, 77]


def test_bulk_edit_is_32_bytes():
    assert L.BULK_EDIT.itemsize == 32
    assert [L.BULK_EDIT.fields[k][1] for k in ("instance", "offset", "length", "reserved", "bytes")] == [0, 4, 6, 7, 8]
    assert L.BULK_EDIT_SPACE == 2900


def test_helper_offsets_are_the_wire_layouts():
    W = L.WIRE_BULK
    off = lambda name: W.fields[name][1]                                        # noqa: E731
    xp, out, eq = W.fields["crosspoints"][0].base, W.fields["outputs"][0].base, W.fields["eq"][0].base
    for side in range(2):
        for o in range(L.WIRE_MAX_OUTPUTS):
            base = off("crosspoints") + (side * L.WIRE_MAX_OUTPUTS + o) * xp.itemsize
            assert L.edit_field(("crosspoints", side, o))[0] == base
            for f in xp.names:
                assert L.edit_field(("crosspoints", side, o, f))[0] == base + xp.fields[f][1]
    for o in range(L.WIRE_MAX_OUTPUTS):
        for f in out.names:
            assert L.edit_field(("outputs", o, f))[0] == off("outputs") + o * out.itemsize + out.fields[f][1]
    for ch in range(L.WIRE_MAX_CHANNELS):
        for b in range(L.MAX_BANDS):
            assert L.edit_field(("eq", ch, b))[0] == off("eq") + (ch * L.MAX_BANDS + b) * eq.itemsize
    for sec in ("global", "crossfeed", "legacy", "leveller", "preamp", "master_volume"):
        sub = W.fields[sec][0]
        for f in sub.names:
            assert L.edit_field((sec, f))[0] == off(sec) + sub.fields[f][1]
    for ch in range(L.WIRE_MAX_CHANNELS):
        assert L.edit_field(("delays", "delay_ms", ch))[0] == off("delays") + 4 * ch
    assert L.edit_field(("preamp", "preamp_db", 1))[0] == off("preamp") + 4
    for f in L.BULK_HOST.names:
        assert L.edit_field(("host", f))[0] == W.itemsize + L.BULK_HOST.fields[f][1]


def test_helper_writes_the_field_bytes():
    e = L.bulk_edit(7, ("eq", 3, 4), (L.PEAKING, (0, 0, 0), 1000.0, 0.7, -4.5))
    assert int(e["instance"][0]) == 7 and int(e["length"][0]) == 16 and int(e["reserved"][0]) == 0
    w = np.zeros(1, L.WIRE_BULK)
    w["eq"][0, 3, 4] = (L.PEAKING, (0, 0, 0), 1000.0, 0.7, -4.5)
    o = int(e["offset"][0])
    assert w.tobytes()[o:o + 16] == e["bytes"][0, :16].tobytes()
    v = L.bulk_edit(0, ("host", "volume_8_8"), -12 * 256)
    assert int(v["offset"][0]) == 2896 and int(v["length"][0]) == 2 and v["bytes"][0, :2].view("<i2")[0] == -12 * 256
    with pytest.raises(ValueError):
        L.bulk_edit(0, ("eq", 11, 0), b"\0")                                     # past the channel rows
    with pytest.raises(ValueError):
        L.bulk_edit(0, ("channel_names",), "x" * 32)                              # 32 bytes: more than one edit carries
