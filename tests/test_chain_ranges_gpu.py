"""GPU: process calls over an instance range, dspi_chain(q)_process_packets_range_* / _process_subframes_range_*.  The bars:
a twin engine fed whole-engine calls (outputs row for row, instance images byte for byte), the engine's own images of the
instances outside the range (unchanged), separate engines holding one clock group each, and the oracle run packet by
packet.  Float engines run in both K1 geometries: 160 instances are 32 mod 64, so in the register-pair geometry
(DSPI_F32_CPL=2) every odd role's rows start half-way into a 64-row group shared with the neighbouring role."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                                  # noqa: E402
from tests.chain_cases import chain_params, chain_params_q28, pcm_bytes                  # noqa: E402
from tests.orc import arm_mute_envelope, make_orc_chain, make_orc_chain_q28             # noqa: E402
from tests.test_chain_packets_gpu import orc_run_packets                                 # noqa: E402

EINVAL, ERANGE = -22, -34
CADENCE = [44] * 9 + [45]                                   # 441 frames every 10 ms
CASES = [("f32f", 1), ("f32f", 2), ("f32s", 1), ("f32s", 2), ("q28", 1)]   # (kind, DSPI_F32_CPL)
KINDS = ["f32f", "f32s", "q28"]


def is_q(kind):
    return kind == "q28"


def pairs(kind):
    return 2 if is_q(kind) else 4


def engine(kind, n, frames=512):
    return api.ChainEngineQ28(n, max_frames=frames) if is_q(kind) else api.ChainEngine(kind, n, max_frames=frames)


def params(oracle, kind, n, fs, seed):
    """Leveller on (look-ahead on most), crossfeed, delays longer than a call, sub on for most instances."""
    P, bq = chain_params_q28(oracle, n, fs, seed) if is_q(kind) else chain_params(oracle, n, fs, seed)
    P["leveller_enabled"] = 1
    P["leveller_lookahead"] = np.arange(n) % 4 != 3
    P["crossfeed_enabled"] = np.arange(n) % 5 != 4
    return P, bq


def tiled(oracle, kind, n, fs, seed):
    """params() for 64 instances, repeated: large engines without a per-instance coefficient computation."""
    P, bq = params(oracle, kind, 64, fs, seed)
    k = -(-n // 64)
    return np.tile(P, k)[:n], np.tile(bq, (k, 1, 1))[:n]


def arm(eng, insts, fs):
    st = np.zeros(1, L.PRESET_MUTE)
    st["smooth_gain"] = 1.0
    api.lib().dspi_preset_mute_arm(st.ctypes.data_as(C.c_void_p), int(fs))
    for i in insts:
        eng.set_preset_mute(st, fs, inst0=int(i))


def setup(eng, P, bq, fs, armed=()):
    eng.set_params(P)
    eng.upload_biquads(bq)
    arm(eng, armed, fs)
    rng = np.random.default_rng(len(P))
    eng.set_spdif_tx(rng.integers(0, 192, len(P)), rng.integers(0, 256, (len(P), 5)).astype(np.uint8))


def call_whole(eng, pcm, bd, frames, subframes):
    return (eng.process_subframes_host if subframes else eng.process_packets_host)(pcm, bd, frames)


def call_range(eng, inst0, pcm, bd, frames, subframes):
    return (eng.process_subframes_range_host if subframes else eng.process_packets_range_host)(inst0, pcm, bd, frames)


def same_rows(got, want, rows):
    """(spdif, pdm, status) of a range call == rows `rows` of a whole-engine call"""
    return (np.array_equal(got[0], want[0][rows]) and np.array_equal(got[1], want[1][rows])
            and got[2].tobytes() == want[2][rows].tobytes())


def snapshot(eng, inst0, n):
    return eng.export_instances(inst0, n), eng.get_spdif_tx(n, inst0).tobytes(), eng.get_preset_mute(n, inst0).tobytes()


def same_snapshot(a, b):
    return np.array_equal(a[0], b[0]) and a[1:] == b[1:]


@pytest.fixture
def libm(oracle):
    oracle.set_libm_f64(1)
    yield oracle
    oracle.set_libm_f64(0)


# mixed tables over the calls; each call alternates words / subframes and 24 / 16-bit input
CALLS = [(CADENCE, 24, False), ([95, 96, 97, 1, 192], 16, True), ([48] * 4, 24, True), ([192, 7, 100], 16, False)]


# ---- 1. pieces equal the whole ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_range_calls_equal_whole_engine_calls(libm, monkeypatch, kind, cpl):
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    n, fs = 160, 48000.0
    ranges = [(0, 64), (64, 128), (128, 160)]
    a, t = engine(kind, n), engine(kind, n)
    try:
        P, bq = params(libm, kind, n, fs, 11)
        for e in (a, t):
            setup(e, P, bq, fs, armed=range(3, n, 7))
        for k, (frames, bd, sub) in enumerate(CALLS):
            pcm = pcm_bytes(n, sum(frames), bd, 100 + k)
            want = call_whole(t, pcm, bd, frames, sub)
            for i0, i1 in ranges:
                got = call_range(a, i0, pcm[i0:i1], bd, frames, sub)
                assert same_rows(got, want, slice(i0, i1)), f"call {k} range [{i0}, {i1})"
        assert np.array_equal(a.export_instances(), t.export_instances())
        assert a.get_spdif_tx().tobytes() == t.get_spdif_tx().tobytes()
        assert a.get_preset_mute().tobytes() == t.get_preset_mute().tobytes()
    finally:
        a.close()
        t.close()


# ---- 2. outside the range nothing changes ---------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_instances_outside_the_range_are_untouched(libm, monkeypatch, kind, cpl):
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    n, fs, i0, m = 224, 48000.0, 64, 81                     # the range ends inside a K1 / K2 group
    a, t = engine(kind, n), engine(kind, n)
    try:
        P, bq = params(libm, kind, n, fs, 21)
        P["host_mute"] = 0
        for i in range(0, n, 3):                            # delay lines longer than one call
            P[i]["matrix"]["outputs"][0]["delay_samples"] = 1500 if i % 2 else 2047
        for e in (a, t):
            setup(e, P, bq, fs, armed=range(0, n, 5))       # armed envelopes inside and outside the range
            call_whole(e, pcm_bytes(n, sum(CADENCE), 24, 22), 24, CADENCE, False)
        before = [snapshot(a, 0, i0), snapshot(a, i0 + m, n - i0 - m)]
        call_range(a, i0, pcm_bytes(m, 481, 16, 23), 16, [95, 96, 97, 1, 192], True)
        after = [snapshot(a, 0, i0), snapshot(a, i0 + m, n - i0 - m)]
        assert all(same_snapshot(x, y) for x, y in zip(before, after))
        pcm = pcm_bytes(n, sum(CADENCE), 24, 24)
        ga, gt = call_whole(a, pcm, 24, CADENCE, False), call_whole(t, pcm, 24, CADENCE, False)
        for rows in (slice(0, i0), slice(i0 + m, n)):
            assert same_rows([x[rows] for x in ga], gt, rows)
        assert np.array_equal(a.export_instances(0, i0), t.export_instances(0, i0))
        assert np.array_equal(a.export_instances(i0 + m, n - i0 - m), t.export_instances(i0 + m, n - i0 - m))
    finally:
        a.close()
        t.close()


# ---- 3. two clocks in one engine ------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_two_clock_groups_share_one_engine(libm, kind):
    """[0, 64) at 44.1 kHz on its cadence, [64, 114) at 96 kHz with feedback-paced 95 / 96 / 97-frame packets, interleaved;
    each group equals an engine holding only that group, and a few instances equal the oracle."""
    na, nb, fa, fb = 64, 50, 44100.0, 96000.0
    Pa, bqa = params(libm, kind, na, fa, 31)
    Pb, bqb = params(libm, kind, nb, fb, 32)
    eng, ea, eb = engine(kind, na + nb), engine(kind, na), engine(kind, nb)
    try:
        eng.set_params(Pa)
        eng.upload_biquads(bqa)
        eng.set_params(Pb, inst0=na)
        eng.upload_biquads(bqb, inst0=na)
        arm(eng, [1, 9], fa)
        arm(eng, [na + 2, na + 40], fb)
        for e, P, bq, fs, armed in ((ea, Pa, bqa, fa, [1, 9]), (eb, Pb, bqb, fb, [2, 40])):
            e.set_params(P)
            e.upload_biquads(bq)
            arm(e, armed, fs)
        mk = make_orc_chain_q28 if is_q(kind) else make_orc_chain
        orc = {0: mk(libm, Pa[0], bqa[0]), 9: mk(libm, Pa[9], bqa[9]), na + 2: mk(libm, Pb[2], bqb[2])}
        arm_mute_envelope(orc[9], fa)
        arm_mute_envelope(orc[na + 2], fb)
        paced = [[96, 97, 96, 95, 96], [97, 97, 96], [95, 96, 96, 97, 95], [96, 96, 95, 96]]
        for k in range(4):
            for inst0, sub_e, n, frames, bd in ((0, ea, na, CADENCE, 24), (na, eb, nb, paced[k], 16)):
                pcm = pcm_bytes(n, sum(frames), bd, 300 + 10 * k + inst0)
                sub = k % 2 == 1
                got = call_range(eng, inst0, pcm, bd, frames, sub)
                want = call_whole(sub_e, pcm, bd, frames, sub)
                assert same_rows(got, want, slice(None)), f"call {k} group at {inst0}"
                for i, ch in orc.items():
                    if inst0 <= i < inst0 + n:
                        ws, wp = orc_run_packets(libm, kind, ch, pcm[i - inst0], bd, frames)
                        if not sub:
                            assert np.array_equal(got[0][i - inst0], ws), f"call {k} instance {i}: S/PDIF words differ from the oracle"
                        if int(ch.out[4 if is_q(kind) else 8].enabled):
                            assert np.array_equal(got[1][i - inst0], wp), f"call {k} instance {i}: PDM differs from the oracle"
        assert np.array_equal(eng.export_instances(0, na), ea.export_instances())
        assert np.array_equal(eng.export_instances(na, nb), eb.export_instances())
    finally:
        for e in (eng, ea, eb):
            e.close()


# ---- 4. ragged and edge ranges ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_ragged_ranges(libm, monkeypatch, kind, cpl):
    """n of 1, 17 and 63, a range in the last 64-block, ends inside K1 / K2 groups; instances no range covers keep their
    images."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    n, fs = 200, 48000.0
    ranges = [(0, 1), (64, 81), (128, 191), (192, 200)]
    covered = np.zeros(n, bool)
    for i0, i1 in ranges:
        covered[i0:i1] = True
    a, t = engine(kind, n), engine(kind, n)
    try:
        P, bq = params(libm, kind, n, fs, 41)
        for e in (a, t):
            setup(e, P, bq, fs, armed=range(0, n, 6))
        initial = a.export_instances()
        for k, (frames, bd, sub) in enumerate(CALLS[:3]):
            pcm = pcm_bytes(n, sum(frames), bd, 400 + k)
            want = call_whole(t, pcm, bd, frames, sub)
            for i0, i1 in ranges:
                assert same_rows(call_range(a, i0, pcm[i0:i1], bd, frames, sub), want, slice(i0, i1)), f"call {k} [{i0}, {i1})"
        got, twin = a.export_instances(), t.export_instances()
        assert np.array_equal(got[covered], twin[covered])
        assert np.array_equal(got[~covered], initial[~covered])
    finally:
        a.close()
        t.close()


@pytest.mark.parametrize("kind", KINDS)
def test_range_in_the_middle_of_8192_instances(oracle, kind):
    n, fs, i0, m = 8192, 48000.0, 4096 - 640, 1000
    frames = [96, 97, 95, 96]
    a, t = engine(kind, n, 384), engine(kind, n, 384)
    try:
        P, bq = tiled(oracle, kind, n, fs, 51)
        for e in (a, t):
            setup(e, P, bq, fs, armed=range(0, n, 37))
        edges = [(i0 - 64, 64), (i0 + m, 64)]
        before = [a.export_instances(s, c) for s, c in edges]
        for k in range(2):
            pcm = pcm_bytes(n, sum(frames), 24, 500 + k)
            want = call_whole(t, pcm, 24, frames, k == 1)
            got = call_range(a, i0, pcm[i0:i0 + m], 24, frames, k == 1)
            assert same_rows(got, want, slice(i0, i0 + m)), f"call {k}"
        assert np.array_equal(a.export_instances(i0, m), t.export_instances(i0, m))
        assert all(np.array_equal(a.export_instances(s, c), b) for (s, c), b in zip(edges, before))
    finally:
        a.close()
        t.close()


# ---- 5. ordering of asynchronous range calls --------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_device_range_calls_are_ordered_on_the_engine_stream(oracle, kind):
    n, fs, F = 192, 48000.0, sum(CADENCE)
    ranges = [(0, 64), (64, 192), (128, 192), (0, 128)]
    a, t = engine(kind, n), engine(kind, n)
    try:
        P, bq = params(oracle, kind, n, fs, 61)
        for e in (a, t):
            setup(e, P, bq, fs, armed=range(0, n, 9))
        pcm = torch.from_numpy(pcm_bytes(n, F, 24, 62)).cuda()
        bufs = {e: [(torch.zeros((i1 - i0, pairs(kind), F, 2), dtype=torch.int32, device="cuda"),
                     torch.zeros((i1 - i0, F, 8), dtype=torch.int32, device="cuda"),
                     torch.zeros((i1 - i0, a._STATUS.itemsize), dtype=torch.uint8, device="cuda")) for i0, i1 in ranges]
                for e in (a, t)}
        torch.cuda.synchronize()
        row = pcm.shape[1]
        for e, synced in ((a, False), (t, True)):
            for (i0, i1), (sp, pd, st) in zip(ranges, bufs[e]):
                e.process_packets_range_device(i0, i1 - i0, pcm.data_ptr() + i0 * row, 24, CADENCE, sp.data_ptr(), pd.data_ptr(), st.data_ptr())
                if synced:
                    e.sync()
        img = a.export_instances()                          # right behind the asynchronous calls
        assert np.array_equal(img, t.export_instances())
        a.sync()
        for x, y in zip(bufs[a], bufs[t]):
            assert all(torch.equal(u, v) for u, v in zip(x, y))
    finally:
        a.close()
        t.close()


# ---- 6. refusals change nothing -----------------------------------------------------------------------------------------
def _raw(eng, name, *args):
    return getattr(api.lib(), eng._PRE + "_" + name)(*args)


@pytest.mark.parametrize("kind", KINDS)
def test_refused_range_calls_change_nothing(oracle, kind):
    n, fs, F = 100, 48000.0, 96
    a = engine(kind, n)
    try:
        P, bq = params(oracle, kind, n, fs, 71)
        setup(a, P, bq, fs, armed=range(0, n, 4))
        a.process_packets_host(pcm_bytes(n, F, 24, 72), 24, [F])
        ref = snapshot(a, 0, n)
        pcm = torch.from_numpy(pcm_bytes(n, F, 24, 73)).cuda()
        sp = torch.full((n * pairs(kind) * F * 4 + 4,), 7, dtype=torch.int32, device="cuda")
        pd = torch.full((n, F, 8), 7, dtype=torch.int32, device="cuda")
        st = torch.full((n, 64), 7, dtype=torch.uint8, device="cuda")
        sp0, pd0, st0 = sp.clone(), pd.clone(), st.clone()
        good = (np.array([F], np.uint16), np.array([F, 0], np.uint16))
        h, p = a._h, C.c_void_p(pcm.data_ptr())
        outs = (C.c_void_p(sp.data_ptr()), C.c_void_p(pd.data_ptr()), C.c_void_p(st.data_ptr()))
        tab = good[0].ctypes.data

        def both(inst0, m, h=h, p=p, nk=1, table=tab, bd=24):
            return tuple(_raw(a, "process_%s_range_device" % form, h, inst0, m, p, bd, nk, table, *outs) for form in ("packets", "subframes"))

        torch.cuda.synchronize()
        assert both(32, 10) == (EINVAL, EINVAL)                                # inst0 not a multiple of 64
        assert both(64, 37) == (ERANGE, ERANGE)                                # past the end
        assert both(0xFFFFFFC0, 0x80) == (ERANGE, ERANGE)                      # end wraps in 32 bits
        assert both(0, 10, p=None) == (EINVAL, EINVAL)                         # NULL pcm
        assert both(0, 10, h=None) == (EINVAL, EINVAL)                         # NULL handle
        assert both(0, 10, nk=2, table=good[1].ctypes.data) == (EINVAL, EINVAL)   # a packet of 0 frames
        assert both(0, 10, nk=0) == (EINVAL, EINVAL)                           # no packets
        assert both(0, 10, table=None) == (EINVAL, EINVAL)                     # no table
        assert both(0, 10, bd=20) == (EINVAL, EINVAL)                          # bit depth
        assert _raw(a, "process_subframes_range_device", h, 0, 10, p, 24, 1, tab, C.c_void_p(sp.data_ptr() + 4), *outs[1:]) == EINVAL   # misaligned subframes
        for name in ("process_packets_range_host", "process_subframes_range_host"):
            assert _raw(a, name, h, 32, 10, p, 24, 1, tab, None, None, None) == EINVAL
            assert _raw(a, name, h, 64, 37, p, 24, 1, tab, None, None, None) == ERANGE
        l0 = a.launch_count
        assert both(64, 0) == (0, 0)                                           # n == 0 does nothing
        assert a.launch_count == l0
        a.sync()
        assert torch.equal(sp, sp0) and torch.equal(pd, pd0) and torch.equal(st, st0)
        assert same_snapshot(snapshot(a, 0, n), ref)
    finally:
        a.close()
