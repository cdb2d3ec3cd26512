"""The chain engines past their staging limits: packet schedules longer than one parameter block of schedule_kernel
(chain_schedule.cuh, kChunk offsets per launch), the preset-mute envelope table regrown on a running engine and its
per-packet lookups over thousands of packets, WireBulkParams applies longer than one staging chunk (bulk_ingest.cuh,
kChunk instances per chunk), and the PDM rows of instances whose sub output is off.  Bars as in test_chain_packets_gpu.py:
S/PDIF words, PDM bits, peaks, clip flags and filter state bit-exact against the oracle run packet by packet, the
leveller's per-block libm in double on both sides (oracle `libm_f64`)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                                          # noqa: E402
from tests.bulk_cases import wire_packet                                                          # noqa: E402
from tests.chain_cases import pcm_bytes                                                           # noqa: E402
from tests.orc import arm_mute_envelope                                                           # noqa: E402
from tests.test_bulk_device_gpu import (audible, bad_packets, expected, host_records, initial, is_q, platform,  # noqa: E402
                                        policy_biquads, replace_records, run_oracle)
from tests.test_chain_packets_gpu import _check_call, _check_filters, _engine, _orc, _params, _sub_on   # noqa: E402
from tests.util import same_bits                                                                  # noqa: E402

FS = 48000.0
N_INST = 9                      # neither a multiple of the 16-instance groups nor of the 4-instance CTAs
OFF_BLOCK = 7936                # offsets per schedule_kernel launch (chain_schedule.cuh kChunk)
BULK_CHUNK = 1024               # instances per staged bulk-ingest chunk (bulk_ingest.cuh kChunk)
SENTINEL = 0x5A5AA5A5


def _sub_output(flavour):
    return 4 if flavour == "q28" else 8


def _set_sub(P, flavour, on):
    for i in range(len(P)):
        P[i]["matrix"]["outputs"][_sub_output(flavour)]["enabled"] = 1 if on[i] else 0


def _lengths(rng, n, choices=(1, 2, 3), long_at=()):
    t = [int(x) for x in rng.choice(choices, n)]
    for p in long_at:
        t[p] = 192
    return t


# ---- 1. schedules past one parameter block ------------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_schedules_past_one_parameter_block(oracle, flavour):
    """7935, 7936 and 7937 packets (one, two and two offset blocks: n packets have n + 1 offsets), about 9000, then 5,
    one engine.  Lengths 1..3 so that offsets and packet indices differ; the only 192-frame packets sit in the second
    block, so the post stage's shared memory and the leveller's block sizes come from it."""
    rng = np.random.default_rng(900)
    calls = [_lengths(rng, OFF_BLOCK - 1), _lengths(rng, OFF_BLOCK), _lengths(rng, OFF_BLOCK + 1, long_at=[OFF_BLOCK]),
             _lengths(rng, 9001, long_at=[OFF_BLOCK, OFF_BLOCK + 3, 8500, 9000]), _lengths(rng, 5)]
    N = N_INST
    P, bq = _params(oracle, flavour, N, FS, 901)
    _set_sub(P, flavour, np.arange(N) % 4 != 2)                 # the sub on most instances
    oracle.set_libm_f64(1)
    eng = _engine(flavour, N, max(sum(c) for c in calls))
    try:
        eng.set_params(P)
        eng.upload_biquads(bq)
        chains = [_orc(oracle, flavour, P[i], bq[i]) for i in range(N)]
        launches = []
        for k, frames in enumerate(calls):
            pcm = pcm_bytes(N, sum(frames), 16, 910 + k)
            n0 = eng.launch_count
            _check_call(oracle, flavour, eng, P, chains, pcm, 16, frames, what=f"call {k} ({len(frames)} packets)")
            launches.append(eng.launch_count - n0)
        _check_filters(flavour, eng, chains)
        # the same slice plan (16 slices) for the three calls: the only difference is the second schedule_kernel launch
        assert launches[1] == launches[0] + 1 and launches[2] == launches[1], launches
    finally:
        eng.close()
        oracle.set_libm_f64(0)


@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_uniform_call_past_one_parameter_block(oracle, flavour):
    """process_host(8000 packets x 2 frames) == process_packets_host([2] * 8000) on a twin: outputs, status, state"""
    n, fpp, N = 8000, 2, N_INST
    P, bq = _params(oracle, flavour, N, FS, 905)
    _set_sub(P, flavour, np.arange(N) % 4 != 2)
    pcm = pcm_bytes(N, n * fpp, 24, 906)
    a, b = _engine(flavour, N, n * fpp), _engine(flavour, N, n * fpp)
    try:
        for e in (a, b):
            e.set_params(P)
            e.upload_biquads(bq)
        ra = a.process_host(pcm, 24, n, fpp)
        rb = b.process_packets_host(pcm, 24, [fpp] * n)
        assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1]) and ra[2].tobytes() == rb[2].tobytes()
        assert np.array_equal(a.state_export(), b.state_export())
        assert a.launch_count == b.launch_count
    finally:
        a.close()
        b.close()


# ---- 2. envelope table regrowth and long searches ----------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_envelope_table_regrowth_and_long_lookups(oracle, flavour):
    """A call without the envelope (no table), then the envelope armed on most instances and calls of 5, 40, 3, ~8000,
    2 and 300 packets: the per-packet volume table grows at the 40- and the 8000-packet call on a running engine.  A
    re-arm right before the long call puts its whole fade-out, hold and fade-in (384 + 512 + 384 samples) inside it; the
    long call ends in 4100 one-frame packets, and the delays of up to MAX - 1 samples put the packet of a delayed sample
    thousands of packets back (the outpost stage's search, and the ring kernel's over the last 4096 frames).  The short
    calls after it read that ring.  Then envelope mode is left and armed again."""
    q = flavour == "q28"
    N = N_INST
    n_out, dmax = (5, 2047) if q else (9, 4095)
    delays = [dmax, 0, dmax - 1, 1, 2000, dmax, 700, dmax - 3, 4000][:n_out]
    rng = np.random.default_rng(920)
    long_call = _lengths(rng, 3900, choices=(1, 2)) + [1] * 4100
    short = {k: _lengths(rng, k, choices=(1, 2)) for k in (5, 40, 3, 2)}
    c300 = _lengths(rng, 300, choices=(1, 2), long_at=[150])
    first = [48, 1, 2, 192, 45, 7]
    F_max = max(sum(long_call), sum(first))
    P, bq = _params(oracle, flavour, N, FS, 921)
    _set_sub(P, flavour, np.arange(N) % 4 != 2)
    for i in range(N):
        P[i]["host_mute"] = 0
        for o in range(n_out):
            P[i]["matrix"]["outputs"][o]["delay_samples"] = delays[(o + i) % n_out]
    armed = [i for i in range(N) if i % 4 != 1]
    oracle.set_libm_f64(1)
    eng = _engine(flavour, N, F_max)
    seed = [930]

    def call(frames, what):
        seed[0] += 1
        _check_call(oracle, flavour, eng, P, chains, pcm_bytes(N, sum(frames), 24, seed[0]), 24, frames, what=what)
        got = eng.get_preset_mute()
        for i in armed:
            if chains[i].mute_env_on:
                assert (int(got[i]["loading"]), int(got[i]["counter"])) == (int(chains[i].preset_loading), int(chains[i].preset_mute_counter)), \
                    f"{what}: instance {i} envelope state"
                assert np.float32(got[i]["smooth_gain"]) == np.float32(chains[i].preset_mute_smooth_gain), f"{what}: instance {i} envelope gain"
        return got

    def arm(states):
        st = np.ascontiguousarray(states).copy()
        for i in armed:
            api.lib().dspi_preset_mute_arm(st[i:i + 1].ctypes.data_as(C.c_void_p), int(FS))
            eng.set_preset_mute(st[i:i + 1], FS, inst0=i)
            arm_mute_envelope(chains[i], FS, smooth_gain=float(chains[i].preset_mute_smooth_gain) if chains[i].mute_env_on else 1.0)

    try:
        eng.set_params(P)
        eng.upload_biquads(bq)
        chains = [_orc(oracle, flavour, P[i], bq[i]) for i in range(N)]
        call(first, "no envelope")
        fresh = np.zeros(N, L.PRESET_MUTE)
        fresh["smooth_gain"] = 1.0
        arm(fresh)
        call(short[5], "5 packets (table allocated)")
        got = call(short[40], "40 packets (table regrown)")
        assert all(int(got[i]["loading"]) == 1 and 0.0 < float(got[i]["smooth_gain"]) < 1.0 for i in armed), "fade-out not under way"
        call(short[3], "3 packets")
        arm(eng.get_preset_mute())                                 # re-arm: the whole envelope inside the long call
        got = call(long_call, f"{len(long_call)} packets (table regrown)")
        assert all(int(got[i]["loading"]) == 0 and float(got[i]["smooth_gain"]) == 1.0 for i in armed), "fade-in not completed"
        call(short[2], "2 packets after the long call")
        call(c300, "300 packets after the long call")
        eng.set_preset_mute(None, FS)                              # leave envelope mode: the constant gain of set_params
        for i in armed:
            chains[i].mute_env_on = 0
            chains[i].preset_mute_gain = float(P[i]["preset_mute_gain"])
        call(short[40], "40 packets, envelope mode left")
        arm(fresh)
        call(c300, "300 packets, armed again")
        _check_filters(flavour, eng, chains)
    finally:
        eng.close()
        oracle.set_libm_f64(0)


# ---- 3. bulk applies past one staging chunk -----------------------------------------------------------------------------
def _custom_crossfeed(kind, fs):
    """a crossfeed record no wire packet of bulk_cases produces (custom preset, fc 1234.5 Hz): every accepted packet
    changes the coefficients, so set_params clears the crossfeed state exactly where the ingest does"""
    if is_q(kind):
        return api.crossfeed_coefficients_q28(fs, True, True, 3, 1234.5, 7.25)
    return api.crossfeed_coefficients(fs, True, True, 3, 1234.5, 7.25)


@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_bulk_apply_past_one_staging_chunk(oracle, kind):
    """2 * 1024 + 37 packets from instance 5 of a 2100-instance engine (a start aligned to neither the 4-instance CTA, the
    32- / 64-channel groups nor the chunk), wire versions mixed, rejected packets at range indices 0, 1023, 1024, 2047,
    2048 and the last one; issued right behind an asynchronous process call."""
    q28 = is_q(kind)
    N, inst0, n = 2100, 5, 2 * BULK_CHUNK + 37
    npk, fpp = 2, 48
    F = npk * fpp
    frames = [fpp] * npk
    sts, P0, bq0 = initial(kind, N, FS, 9300)
    P0["crossfeed"] = _custom_crossfeed(kind, FS)
    packets = np.concatenate([audible(wire_packet(platform(kind), 9400 + k, version=2 + k % 5)) for k in range(n)])
    edges = [0, BULK_CHUNK - 1, BULK_CHUNK, 2 * BULK_CHUNK - 1, 2 * BULK_CHUNK, n - 1]
    bad = bad_packets(kind)
    for j, k in enumerate(edges):
        packets[k] = bad[1 + j % 7]
    hv = host_records(n, 9401)
    pcm = pcm_bytes(N, 2 * F, 24, 9402)
    c0, c1 = np.ascontiguousarray(pcm[:, :F * 6]), np.ascontiguousarray(pcm[:, F * 6:])
    pairs, status_t = (2, L.STATUS_Q28) if q28 else (4, L.STATUS)
    sub_o = 4 if q28 else 8
    freqs = np.geomspace(20.0, 20000.0, 12).astype(np.float32)
    oracle.set_libm_f64(1)
    eng, twin = _engine(kind, N, F), _engine(kind, N, F)
    try:
        for e in (eng, twin):
            e.set_params(P0)
            e.upload_biquads(bq0)
        r0 = twin.process_packets_host(c0, 24, frames)
        d_pcm = torch.from_numpy(c0).cuda()
        sp = torch.zeros((N, pairs, F, 2), dtype=torch.int32, device="cuda")
        pd = torch.zeros((N, F, 8), dtype=torch.int32, device="cuda")
        stt = torch.zeros((N * status_t.itemsize,), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        eng.process_packets_device(d_pcm.data_ptr(), 24, frames, sp.data_ptr(), pd.data_ptr(), stt.data_ptr())
        res = eng.apply_bulk_device(packets, FS, inst0=inst0, host=hv)          # no sync in between
        eng.sync()
        # the call in flight finished on the old records
        assert np.array_equal(sp.cpu().numpy(), r0[0]), "in-flight call: S/PDIF words"
        assert np.array_equal(pd.cpu().numpy().view(np.uint32), r0[1]), "in-flight call: PDM bits"
        assert stt.cpu().numpy().tobytes() == r0[2].tobytes(), "in-flight call: status"

        base = twin.download_biquads()                                          # the state the call left
        got = eng.download_biquads()
        Pt, bqt = P0.copy(), base.copy()
        for k in range(n):
            i = inst0 + k
            rc, P = expected(oracle, sts[i], packets[k:k + 1], FS, hv[k], False)
            assert int(res[k]) == rc, f"range index {k}: result code {int(res[k])}, want {rc}"
            if rc == 0:
                P["preset_mute_gain"] = P0[i]["preset_mute_gain"]                 # left alone by the call
                Pt[i] = P[0]
                bqt[i] = policy_biquads(oracle, q28, sts[i], base[i], FS)
        assert sorted(int(k) for k in np.flatnonzero(res)) == edges
        for i in range(N):
            assert same_bits(got[i], bqt[i]), f"instance {i}: biquads (range index {i - inst0})"

        twin.set_params(Pt)
        twin.upload_biquads(bqt)
        assert np.array_equal(eng.response(freqs, FS).view(np.uint32), twin.response(freqs, FS).view(np.uint32)), "parameter rows"
        a, b = eng.process_packets_host(c1, 24, frames), twin.process_packets_host(c1, 24, frames)
        sub = np.array([bool(Pt[i]["matrix"]["outputs"][sub_o]["enabled"]) for i in range(N)])
        assert np.array_equal(a[0], b[0]), "S/PDIF words against the twin"
        assert sub.any() and np.array_equal(a[1][sub], b[1][sub]), "PDM bits against the twin"
        assert a[2].tobytes() == b[2].tobytes(), "status against the twin"
        # filter state field by field (the state blob holds the biquad records with their padding bytes)
        assert same_bits(eng.download_biquads(), twin.download_biquads()), "filter state against the twin"

        # both sides of every chunk edge (and of the range) against the oracle, continued from the first call
        near = sorted({inst0 + k + d for k in edges for d in (-1, 0, 1)} | {inst0 - 1, inst0 + n})
        for i in near:
            ch = _orc(oracle, kind, P0[i], bq0[i])
            run_oracle(oracle, kind, ch, c0[i], 24, npk, fpp)
            k = i - inst0
            if 0 <= k < n and res[k] == 0:
                ch = replace_records(oracle, ch, Pt[i:i + 1], sts[i], FS, q28)
            ws, wp = run_oracle(oracle, kind, ch, c1[i], 24, npk, fpp)
            assert np.array_equal(a[0][i], ws), f"instance {i} (range index {k}): S/PDIF words"
            if sub[i]:
                assert np.array_equal(a[1][i], wp), f"instance {i} (range index {k}): PDM bits"
            assert list(a[2][i]["peaks"]) == list(ch.peaks)[:len(a[2][i]["peaks"])], f"instance {i}: meters"

        # one more instance than a chunk takes a second round of staging launches; a third chunk costs as much again
        counts = []
        for m in (BULK_CHUNK, BULK_CHUNK + 1, n):
            l0 = eng.launch_count
            eng.apply_bulk_device(packets[:m], FS, inst0=inst0, host=hv[:m])
            counts.append(eng.launch_count - l0)
        assert counts[1] > counts[0] and counts[2] - counts[1] == counts[1] - counts[0], counts
    finally:
        eng.close()
        twin.close()
        oracle.set_libm_f64(0)


# ---- 4. PDM rows of instances without a sub -----------------------------------------------------------------------------
def _bulk_sub_packets(flavour, on):
    """one wire packet per instance, the sub output (the last one) enabled where ``on``"""
    out = []
    for i in range(len(on)):
        w = audible(wire_packet(platform(flavour), 9500 + i))
        w["outputs"][0]["enabled"][_sub_output(flavour)] = 1 if on[i] else 0
        w["outputs"][0]["mute"][_sub_output(flavour)] = 0
        out.append(w)
    return np.concatenate(out)


@pytest.mark.parametrize("route", ["set_params", "bulk", "fixed"])
@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_pdm_rows_of_sub_less_instances(oracle, flavour, route):
    """The sub on everywhere for call 1, then off on odd instances (through set_params or apply_bulk_device) for a call
    of the same length and a shorter one; or ("fixed") off on odd instances from the start, with calls getting shorter.
    The _host forms (words and subframes) return all-zero rows for sub-less instances; the _device form leaves the
    caller's rows of those instances untouched.  Rows of instances with a sub are the same in all three."""
    N = N_INST
    calls = [[48] * 6, [48] * 6, [48, 45, 1, 2]] if route != "fixed" else [[48] * 6, [48] * 4 + [7], [45, 1, 2]]
    F_max = max(sum(c) for c in calls)
    odd = np.arange(N) % 2 == 1
    P, bq = _params(oracle, flavour, N, FS, 940)
    _set_sub(P, flavour, ~odd if route == "fixed" else np.ones(N, bool))
    words, subf, dev = engs = [_engine(flavour, N, F_max) for _ in range(3)]
    pairs = 2 if flavour == "q28" else 4
    try:
        for e in engs:
            e.set_params(P)
            e.upload_biquads(bq)
        on = np.array([_sub_on(flavour, P[i]) for i in range(N)])
        for k, frames in enumerate(calls):
            if k == 1 and route == "set_params":
                _set_sub(P, flavour, ~odd)
                for e in engs:
                    e.set_params(P)
                on = ~odd
            elif k == 1 and route == "bulk":
                packets = _bulk_sub_packets(flavour, ~odd)
                for e in engs:
                    assert not e.apply_bulk_device(packets, FS).any()
                on = ~odd
            F = sum(frames)
            pcm = pcm_bytes(N, F, 16, 941 + k)
            sw, pw, _ = words.process_packets_host(pcm, 16, frames)
            _, ps, _ = subf.process_subframes_host(pcm, 16, frames)
            d_pcm = torch.from_numpy(pcm).cuda()
            sp = torch.zeros((N, pairs, F, 2), dtype=torch.int32, device="cuda")
            pd = torch.full((N, F, 8), SENTINEL, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            dev.process_packets_device(d_pcm.data_ptr(), 16, frames, sp.data_ptr(), pd.data_ptr(), 0)
            dev.sync()
            pdv = pd.cpu().numpy().view(np.uint32)
            what = f"{route}, call {k} ({F} frames)"
            assert on.any() and all(pw[i].any() for i in np.flatnonzero(on)), f"{what}: a sub's PDM rows are empty"
            assert np.array_equal(pw[on], ps[on]) and np.array_equal(pw[on], pdv[on]), f"{what}: PDM rows of instances with a sub"
            assert np.array_equal(sw, sp.cpu().numpy()), f"{what}: S/PDIF words host vs device"
            for i in np.flatnonzero(~on):
                assert not pw[i].any(), f"{what}: instance {i} (no sub): PDM rows of the words host form not zero"
                assert not ps[i].any(), f"{what}: instance {i} (no sub): PDM rows of the subframes host form not zero"
                assert (pdv[i] == SENTINEL).all(), f"{what}: instance {i} (no sub): the device form wrote its PDM rows"
    finally:
        for e in engs:
            e.close()
