"""Per-packet schedules (dspi_chain(q)_process_packets_*): calls whose USB packets have different lengths - the 44.1 kHz
cadence, feedback-paced streams, mixed 1..192-frame packets - against the oracle run packet by packet with each packet's
own byte length (usb_audio.c:500 / :968).  Bars as in test_chain_gpu.py: S/PDIF words, PDM bits, peaks, clip flags and
filter state bit-exact, the leveller's per-block libm in double on both sides (oracle `libm_f64`)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                                 # noqa: E402
from tests.chain_cases import chain_params, chain_params_q28, pcm_bytes                  # noqa: E402
from tests.orc import RefChain, RefPdm, arm_mute_envelope, make_orc_chain, make_orc_chain_q28  # noqa: E402

CADENCE_44K1 = [44] * 9 + [45]                       # 441 frames every 10 ms


def _engine(flavour, N, F):
    return api.ChainEngineQ28(N, max_frames=F) if flavour == "q28" else api.ChainEngine(flavour, N, max_frames=F)


def _params(oracle, flavour, N, fs, seed, leveller=True, lookahead=True):
    P, bq = chain_params_q28(oracle, N, fs, seed) if flavour == "q28" else chain_params(oracle, N, fs, seed)
    if leveller:
        P["leveller_enabled"] = 1
        if lookahead:
            P["leveller_lookahead"] = np.arange(N) % 4 != 3          # look-ahead on most instances
    else:
        P["leveller_enabled"] = 0
    return P, bq


def _orc(oracle, flavour, P, bq):
    return make_orc_chain_q28(oracle, P, bq) if flavour == "q28" else make_orc_chain(oracle, P, bq)


def orc_run_packets(oracle, flavour, chain, pcm, bit_depth, frames):
    """The oracle, one process_audio_packet() per entry of ``frames`` with that packet's own byte length;
    returns (spdif [pairs, F, 2], pdm [F, 8])."""
    F, bpf = int(sum(frames)), (6 if bit_depth == 24 else 4)
    spdif = np.zeros((2 if flavour == "q28" else 4, F, 2), np.int32)
    pdm = np.zeros((F, 8), np.uint32)
    fn = getattr(oracle.lib, "orc_q28_chain_packet" if flavour == "q28" else f"orc_{flavour}_chain_packet")
    data = np.ascontiguousarray(pcm)
    f0 = 0
    for k in frames:
        fn(C.addressof(chain), data.ctypes.data + f0 * bpf, int(k) * bpf, bit_depth, spdif.ctypes.data + f0 * 8, F * 2, pdm.ctypes.data + f0 * 32)
        f0 += int(k)
    return spdif, pdm


def _sub_on(flavour, p):
    return bool(p["matrix"]["outputs"][4 if flavour == "q28" else 8]["enabled"])


def _check_call(oracle, flavour, eng, P, chains, pcm, bit_depth, frames, what=""):
    spdif, pdm, status = eng.process_packets_host(pcm, bit_depth, frames)
    for i in range(len(chains)):
        ws, wp = orc_run_packets(oracle, flavour, chains[i], pcm[i], bit_depth, frames)
        assert np.array_equal(spdif[i], ws), f"{what} instance {i}: S/PDIF words differ"
        if _sub_on(flavour, P[i]):
            assert np.array_equal(pdm[i], wp), f"{what} instance {i}: PDM bitstream differs"
        n_roles = len(status[i]["peaks"])
        assert list(status[i]["peaks"]) == list(chains[i].peaks)[:n_roles], f"{what} instance {i}: peaks"
        assert int(status[i]["clip_flags"]) == int(chains[i].clip_flags), f"{what} instance {i}: clip flags"
    return spdif, pdm, status


def _check_filters(flavour, eng, chains):
    got = eng.download_biquads()
    for i, ch in enumerate(chains):
        if flavour == "q28":
            for r in range(7):
                want = np.frombuffer(bytes(ch.filters[r]), L.BIQUAD_Q28)
                assert np.array_equal(got[i, r]["s1"], want["s1"]) and np.array_equal(got[i, r]["s2"], want["s2"]), f"instance {i} role {r}: state"
        else:
            want = np.frombuffer(bytes(ch.filters), L.BIQUAD_F32).reshape(11, 12)
            for name in ("s1", "s2", "svic1eq", "svic2eq"):
                assert np.array_equal(got[i][name].view(np.uint32), want[name].view(np.uint32)), f"instance {i}: filter state {name}"


def _run(oracle, flavour, N, fs, bit_depth, calls, seed, leveller=True):
    """``calls``: one packet-length list per process call.  Engine and oracle side by side, call after call."""
    F_max = max(int(sum(c)) for c in calls)
    P, bq = _params(oracle, flavour, N, fs, seed, leveller=leveller)
    bpf = 6 if bit_depth == 24 else 4
    pcm = pcm_bytes(N, sum(int(sum(c)) for c in calls), bit_depth, seed + 1)
    oracle.set_libm_f64(1)
    eng = _engine(flavour, N, F_max)
    try:
        eng.set_params(P)
        eng.upload_biquads(bq)
        chains = [_orc(oracle, flavour, P[i], bq[i]) for i in range(N)]
        f0 = 0
        for k, frames in enumerate(calls):
            F = int(sum(frames))
            chunk = np.ascontiguousarray(pcm[:, f0 * bpf:(f0 + F) * bpf])
            _check_call(oracle, flavour, eng, P, chains, chunk, bit_depth, frames, what=f"call {k}")
            f0 += F
        _check_filters(flavour, eng, chains)
    finally:
        eng.close()
        oracle.set_libm_f64(0)


# ---- 1. the 44.1 kHz cadence ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bit_depth", [16, 24])
@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_44k1_cadence(oracle, flavour, bit_depth):
    """nine 44-frame packets and one of 45, 23 packets (2.3 cadences) in one call, then 17 more in a second call"""
    sched = CADENCE_44K1 * 4
    _run(oracle, flavour, N=40, fs=44100.0, bit_depth=bit_depth, calls=[sched[:23], sched[23:]], seed=700)


# ---- 2. feedback-paced and mixed lengths ------------------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_feedback_paced_lengths(oracle, flavour):
    rng = np.random.default_rng(710)
    calls = [list(rng.integers(47, 50, 21)), list(rng.integers(47, 50, 13))]
    _run(oracle, flavour, N=35, fs=48000.0, bit_depth=16, calls=calls, seed=711)


@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_mixed_packet_lengths_in_one_call(oracle, flavour):
    """1-, 2-, 45- and 192-frame packets side by side: the leveller's count == 1 case, its ramp over count - 1, and the
    post stage's shared memory sized by the longest packet"""
    calls = [[1, 2, 45, 192, 2, 1, 192, 45, 1, 1, 2, 192], [192, 1, 45, 2]]
    _run(oracle, flavour, N=33, fs=48000.0, bit_depth=24, calls=calls, seed=720)


# ---- 3. preset-mute envelope over packets of different lengths ------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_envelope_fade_over_variable_packets(oracle, flavour):
    """A preset mute armed on most instances at 48 kHz: the 384-sample fade-out, the 512-sample hold and the fade-in step
    by each packet's own length; the hold ends inside the second call's 192-frame packet and the fade-in runs on into the
    third call.  The delays put T - dl into earlier, shorter packets of the same call (the per-packet gain of the delayed
    sample is looked up by frame, not by T / fpp)."""
    fs = 48000.0
    N = 12
    calls = [[7, 44, 1, 96, 45, 2, 192, 33, 48, 9], [1, 192, 47, 3, 96, 5], [45, 60, 2, 192, 96, 1]]
    n_out = 5 if flavour == "q28" else 9
    delays = [0, 1, 3, 46, 52, 101, 180, 250, 700][:n_out]
    F_max = max(sum(c) for c in calls)
    P, bq = _params(oracle, flavour, N, fs, 730)
    for i in range(N):
        P[i]["host_mute"] = 0
        for o in range(n_out):
            P[i]["matrix"]["outputs"][o]["delay_samples"] = delays[(o + i) % n_out]
    armed = [i for i in range(N) if i % 4 != 1]
    pcm = pcm_bytes(N, sum(sum(c) for c in calls), 24, 731)
    oracle.set_libm_f64(1)
    eng = _engine(flavour, N, F_max)
    try:
        eng.set_params(P)
        eng.upload_biquads(bq)
        chains = [_orc(oracle, flavour, P[i], bq[i]) for i in range(N)]
        st = np.zeros(len(armed), L.PRESET_MUTE)
        st["smooth_gain"] = 1.0
        for k, i in enumerate(armed):
            api.lib().dspi_preset_mute_arm(st[k:k + 1].ctypes.data_as(C.c_void_p), int(fs))
            eng.set_preset_mute(st[k:k + 1], fs, inst0=i)
            arm_mute_envelope(chains[i], fs)
        f0 = 0
        for k, frames in enumerate(calls):
            chunk = np.ascontiguousarray(pcm[:, f0 * 6:(f0 + sum(frames)) * 6])
            f0 += sum(frames)
            _check_call(oracle, flavour, eng, P, chains, chunk, 24, frames, what=f"call {k}")
            got = eng.get_preset_mute()
            for i in armed:
                assert (int(got[i]["loading"]), int(got[i]["counter"])) == (int(chains[i].preset_loading), int(chains[i].preset_mute_counter))
                assert np.float32(got[i]["smooth_gain"]) == np.float32(chains[i].preset_mute_smooth_gain)
            if k == 0:
                assert all(int(got[i]["loading"]) == 1 and float(got[i]["smooth_gain"]) == 0.0 for i in armed), "hold not reached"
            if k == 1:
                assert all(int(got[i]["loading"]) == 0 and 0.0 < float(got[i]["smooth_gain"]) < 1.0 for i in armed), "fade-in not under way"
        assert all(float(got[i]["smooth_gain"]) == 1.0 for i in armed)
        _check_filters(flavour, eng, chains)
    finally:
        eng.close()
        oracle.set_libm_f64(0)


# ---- 4. a call longer than the delay ring ------------------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_call_longer_than_the_delay_ring(oracle, flavour):
    """> 4096 (float) / > 2048 (Q28) frames of feedback-paced packets per call, two calls"""
    rng = np.random.default_rng(740)
    n = 48 if flavour != "q28" else 24
    calls = [list(rng.integers(95, 98, n)), list(rng.integers(95, 98, n))]
    assert min(sum(c) for c in calls) > (4096 if flavour != "q28" else 2048)
    _run(oracle, flavour, N=6, fs=96000.0, bit_depth=16, calls=calls, seed=741)


# ---- 5. one schedule split over calls --------------------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_split_schedule_gives_the_same_bytes(oracle, flavour):
    """the same packets in one call and in three calls: identical words, PDM bits, meters and state, both equal to the oracle"""
    rng = np.random.default_rng(750)
    sched = [int(x) for x in rng.choice([1, 44, 45, 47, 48, 49, 96, 192], 30)]
    parts = [sched[:7], sched[7:19], sched[19:]]
    N, bit_depth, fs = 20, 24, 48000.0
    F = sum(sched)
    P, bq = _params(oracle, flavour, N, fs, 751)
    pcm = pcm_bytes(N, F, bit_depth, 752)
    oracle.set_libm_f64(1)
    one, three = _engine(flavour, N, F), _engine(flavour, N, F)
    try:
        for e in (one, three):
            e.set_params(P)
            e.upload_biquads(bq)
        chains = [_orc(oracle, flavour, P[i], bq[i]) for i in range(N)]
        s1, p1, st1 = _check_call(oracle, flavour, one, P, chains, pcm, bit_depth, sched, what="one call")
        outs, f0 = [], 0
        for frames in parts:
            n = sum(frames)
            outs.append(three.process_packets_host(np.ascontiguousarray(pcm[:, f0 * 6:(f0 + n) * 6]), bit_depth, frames))
            f0 += n
        assert np.array_equal(s1, np.concatenate([o[0] for o in outs], axis=2))
        sub = np.array([_sub_on(flavour, P[i]) for i in range(N)])        # PDM rows are written for instances with a sub only
        assert sub.any() and np.array_equal(p1[sub], np.concatenate([o[1] for o in outs], axis=1)[sub])
        assert st1.tobytes() == outs[-1][2].tobytes()
        assert np.array_equal(one.state_export(), three.state_export())
        _check_filters(flavour, three, chains)
    finally:
        one.close()
        three.close()
        oracle.set_libm_f64(0)


# ---- 6. a uniform table is the frames_per_packet call --------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_uniform_table_equals_frames_per_packet(oracle, flavour):
    """n equal lengths through process_packets_* == process_* with frames_per_packet: outputs, status and the state blob,
    host and device forms, over two calls"""
    N, n_packets, fpp, fs = 36, 9, 96, 96000.0
    F = n_packets * fpp
    P, bq = _params(oracle, flavour, N, fs, 760)
    pcm = pcm_bytes(N, 2 * F, 24, 761)
    engs = [_engine(flavour, N, F) for _ in range(4)]
    try:
        for e in engs:
            e.set_params(P)
            e.upload_biquads(bq)
        pairs = 2 if flavour == "q28" else 4
        status_t = L.STATUS_Q28 if flavour == "q28" else L.STATUS
        for call in range(2):
            chunk = np.ascontiguousarray(pcm[:, call * F * 6:(call + 1) * F * 6])
            a = engs[0].process_host(chunk, 24, n_packets, fpp)
            b = engs[1].process_packets_host(chunk, 24, [fpp] * n_packets)
            d_pcm = torch.from_numpy(chunk).cuda()
            dev = []
            for e, packets in ((engs[2], False), (engs[3], True)):
                sp = torch.zeros((N, pairs, F, 2), dtype=torch.int32, device="cuda")
                pd = torch.zeros((N, F, 8), dtype=torch.int32, device="cuda")
                stt = torch.zeros((N * status_t.itemsize,), dtype=torch.uint8, device="cuda")
                if packets:
                    e.process_packets_device(d_pcm.data_ptr(), 24, np.full(n_packets, fpp), sp.data_ptr(), pd.data_ptr(), stt.data_ptr())
                else:
                    e.process_device(d_pcm.data_ptr(), 24, n_packets, fpp, sp.data_ptr(), pd.data_ptr(), stt.data_ptr())
                e.sync()
                dev.append((sp.cpu().numpy(), pd.cpu().numpy().view(np.uint32), stt.cpu().numpy()))
            for k in range(2):
                assert np.array_equal(a[k], b[k]), f"call {call}: host output {k}"
                assert np.array_equal(dev[0][k], dev[1][k]), f"call {call}: device output {k}"
                assert np.array_equal(a[k], dev[0][k]), f"call {call}: host vs device output {k}"
            assert a[2].tobytes() == b[2].tobytes() == dev[0][2].tobytes() == dev[1][2].tobytes()
        blobs = [e.state_export() for e in engs]
        assert all(np.array_equal(blobs[0], x) for x in blobs[1:])
    finally:
        for e in engs:
            e.close()


# ---- 7. the compiled reference ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bit_depth", [16, 24])
@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_44k1_cadence_equals_compiled_reference(oracle, flavour, bit_depth):
    """the reference's own process_audio_packet() with data_len = 44 or 45 frames; leveller off, as in
    test_chain_ref_gpu.py (its per-block libm is the one policy item)"""
    if not (RefChain.available() and RefPdm.available()):
        pytest.skip("oracle/_ref chain builds not present")
    ref, ref_pdm = RefChain(flavour), RefPdm()
    fs, N = 44100.0, 24
    frames = (CADENCE_44K1 * 3)[:23]
    F, bpf = sum(frames), (6 if bit_depth == 24 else 4)
    P, bq = _params(oracle, flavour, N, fs, 770, leveller=False)
    P["preset_mute_gain"] = 1.0
    pcm = pcm_bytes(N, F, bit_depth, 771)
    eng = _engine(flavour, N, F)
    try:
        eng.set_params(P)
        eng.upload_biquads(bq)
        spdif, pdm, status = eng.process_packets_host(pcm, bit_depth, frames)
        for i in range(N):
            ch = _orc(oracle, flavour, P[i], bq[i])
            ws = np.zeros((ref.n_pairs, F, 2), np.int32)
            sub = np.zeros(F, np.int32)
            got, f0, tot = C.c_uint32(), 0, 0
            data = np.ascontiguousarray(pcm[i])
            for k in frames:
                n = ref.lib.ref_chain_packet(C.addressof(ch), int(fs), data.ctypes.data + f0 * bpf, k * bpf, bit_depth,
                                             ws.ctypes.data + f0 * 8, F * 2, sub.ctypes.data + tot * 4, C.byref(got))
                assert n == k, f"reference returned {n:#x}"
                f0 += k
                tot += got.value
            assert np.array_equal(spdif[i], ws), f"instance {i}: S/PDIF words differ from the compiled reference"
            if _sub_on(flavour, P[i]):
                words, _ = ref_pdm.run(sub[:tot])
                assert np.array_equal(pdm[i], words), f"instance {i}: PDM bits differ from the compiled reference"
            assert list(status[i]["peaks"]) == list(ch.peaks)[:len(status[i]["peaks"])]
            assert int(status[i]["clip_flags"]) == int(ch.clip_flags)
    finally:
        eng.close()


# ---- 8. argument validation --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_packet_tables_are_validated(flavour):
    eng = _engine(flavour, 4, 100)
    pre = "dspi_chainq" if flavour == "q28" else "dspi_chain"
    host, dev = getattr(api.lib(), pre + "_process_packets_host"), getattr(api.lib(), pre + "_process_packets_device")
    try:
        pcm = np.zeros((4, 100 * 6), np.uint8)
        d_pcm = torch.zeros(4 * 100 * 6, dtype=torch.uint8, device="cuda")
        launches = eng.launch_count
        for fn, ptr in ((host, pcm.ctypes.data), (dev, d_pcm.data_ptr())):
            def call(table, n=None, bit_depth=24):
                t = None if table is None else np.ascontiguousarray(table, np.uint16)
                return fn(eng._h, C.c_void_p(ptr), bit_depth, len(table) if n is None else n, None if t is None else t.ctypes.data, None, None, None)
            assert call(None, n=2) == -22
            assert call([48, 48], n=0) == -22
            assert call([48, 0, 48]) == -22
            assert call([48, 193]) == -22
            assert call([48, 48], bit_depth=20) == -22
            assert call([96, 5]) == -34                          # 101 frames > max_frames 100
            assert call([96, 4]) == 0                             # exactly max_frames
        eng.sync()
        assert eng.launch_count > launches
        with pytest.raises(api.DspiError):
            eng.process_packets_host(np.zeros((4, 0), np.uint8), 24, [])
        with pytest.raises(api.DspiError):
            eng.process_packets_host(np.zeros((4, 65537 * 6), np.uint8), 24, [65537])
    finally:
        eng.close()
