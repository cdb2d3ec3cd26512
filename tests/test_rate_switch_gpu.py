"""GPU: dspi_chain(q)_set_rate_device - perform_rate_change() (main.c:132-171) for many instances, each at its own rate,
re-derived on the device from the configuration record (bulk_ingest.cuh rate_kernel).  The expected engines come from
the pinned pieces of test_bulk_device_gpu.py: dspi_bulk_params_apply for the state, the oracle's generators under the libm
policy for the derived records, and a twin engine configured directly at the new rate."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                          # noqa: E402
from tests.bulk_cases import wire_packet                                          # noqa: E402
from tests.chain_cases import pcm_bytes                                           # noqa: E402
from tests.orc import make_orc_chain, make_orc_chain_q28                           # noqa: E402
from tests.test_bulk_device_gpu import (audible, engine, expected, host_records, initial, is_q, platform, policy_biquads,   # noqa: E402
                                        replace_records, run_oracle)
from tests.test_preset_device_gpu import fixture                                  # noqa: E402
from tests.util import same_bits                                                  # noqa: E402

KINDS = ["f32f", "f32s", "q28"]
EINVAL, ERANGE = -22, -34
CURRENT, STALE, UNSET = L.BULK_CURRENT, L.BULK_STALE, L.BULK_UNSET
CHUNK = 1024                                                                      # bulk::kChunk


def roles(kind):
    return 7 if is_q(kind) else 11


def packets_for(kind, n, seed, fmax=None, versions=(2, 3, 4, 5, 6)):
    """audible packets of the given format versions; with fmax, every recipe below it (so no clamp depends on the rate)"""
    w = np.concatenate([audible(wire_packet(platform(kind), seed + i, version=versions[i % len(versions)])) for i in range(n)])
    if fmax is not None:
        w["eq"]["freq"] = np.minimum(w["eq"]["freq"], np.float32(fmax))
    return w


def record_state(oracle, kind, st, fs):
    """``st`` with its recipes clamped as dsp_compute_coefficients() at ``fs`` writes them back: what the record holds"""
    out = st.copy()
    rec = np.ascontiguousarray(out[0]["recipes"][:roles(kind)]).copy()
    bq = np.zeros(rec.shape, L.BIQUAD_Q28 if is_q(kind) else L.BIQUAD_F32)
    oracle.eq_coeffs(is_q(kind), rec, bq, fs)
    out[0]["recipes"][:roles(kind)] = rec
    return out


def configured(oracle, kind, n, fs, seed, hv, fmax=None):
    """An engine of n instances configured by apply_bulk_device at fs on top of a host-route configuration (preset-mute gain
    1, so the outputs are audible), and its oracle chains: (engine, packets, applied states, chains)."""
    q28 = is_q(kind)
    sts, P0, bq0 = initial(kind, n, fs, seed)
    packets = packets_for(kind, n, seed + 500, fmax)
    eng = engine(kind, n, 384)
    eng.set_params(P0)
    eng.upload_biquads(bq0)
    assert not eng.apply_bulk_device(packets, fs, host=hv).any()
    chains = []
    for i in range(n):
        rc, P = expected(oracle, sts[i], packets[i:i + 1], fs, hv[i], False)
        assert rc == 0
        P["preset_mute_gain"] = P0[i]["preset_mute_gain"]
        chains.append((make_orc_chain_q28 if q28 else make_orc_chain)(oracle, P[0], policy_biquads(oracle, q28, sts[i], bq0[i], fs)))
    return eng, packets, sts, P0, chains


def switched(oracle, kind, chain, st, w, hv, pmg, fs_old, fs_new):
    """The oracle chain of an instance after the switch: gains as before (the same packet gives the same gains at any rate),
    every rate-dependent record at fs_new, filters from the record's recipes (clamped at fs_old), running state kept except
    the crossfeed's."""
    rc, P = expected(oracle, st.copy(), w, fs_new, hv, False)
    assert rc == 0
    P["preset_mute_gain"] = pmg
    return replace_records(oracle, chain, P, record_state(oracle, kind, st, fs_old), fs_new, is_q(kind))


def outputs_match(oracle, kind, eng, chains, packets, pcm, npk, fpp, what=""):
    """one process call against the oracle chains: S/PDIF words, PDM bits of instances whose sub is on, meters"""
    spdif, pdm, status = eng.process_host(pcm, 24, npk, fpp)
    sub = roles(kind) - 3
    for i, ch in enumerate(chains):
        ws, wp = run_oracle(oracle, kind, ch, pcm[i], 24, npk, fpp)
        assert np.array_equal(spdif[i], ws), f"{what} instance {i}: S/PDIF words"
        if packets[i]["outputs"]["enabled"][sub]:
            assert np.array_equal(pdm[i], wp), f"{what} instance {i}: PDM bits"
        assert list(status[i]["peaks"]) == list(ch.peaks)[:len(status[i]["peaks"])], f"{what} instance {i}: meters"


@pytest.fixture
def libm(oracle):
    oracle.set_libm_f64(1)
    yield oracle
    oracle.set_libm_f64(0)


# ---- 1. coefficients against the oracle policy, state kept except on flips ------------------------------------------------
@pytest.mark.parametrize("rates", [(96000.0, 44100.0), (44100.0, 96000.0), (48000.0, 88200.0)])
@pytest.mark.parametrize("kind", KINDS)
def test_coefficients_match_the_oracle_policy(libm, kind, rates):
    oracle, q28 = libm, is_q(kind)
    A, B = rates
    n, npk, fpp = 37, 2, 96                                    # neither a multiple of 32 nor of the CTA's 4 instances
    hv = host_records(n, 7)
    eng, packets, sts, _, _ = configured(oracle, kind, n, A, 1000, hv)
    try:
        eng.process_host(pcm_bytes(n, npk * fpp, 24, 11), 24, npk, fpp)          # running state in every band
        base = eng.download_biquads()
        res = eng.set_rate_device(np.full(n, B, np.float32))
        assert (res == CURRENT).all()
        got = eng.download_biquads()
        for i in range(n):
            want = policy_biquads(oracle, q28, record_state(oracle, kind, sts[i], A), base[i], B)
            assert same_bits(got[i], want), f"instance {i}"
        if not q28:
            live = base["bypass"] == 0
            up, down = (got["use_svf"] > base["use_svf"]) & live, (got["use_svf"] < base["use_svf"]) & live
            assert (up.any() if B > A else down.any()), "bands that flip topology"
            assert (base["s1"][up | down] != 0).any() or (base["svic1eq"][up | down] != 0).any(), "flipped bands had state"
    finally:
        eng.close()


# ---- 2. a running engine continues like the main loop -----------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_running_engine_continues_like_the_main_loop(libm, kind):
    oracle = libm
    N, inst0, n, npk, fpp, A = 13, 3, 7, 4, 96, 96000.0
    F = npk * fpp
    rates = np.array([44100.0, 48000.0, 88200.0, 192000.0, 44100.0, 32000.0, 96000.0], np.float32)
    hv = host_records(N, 22)
    eng, packets, sts, P0, chains = configured(oracle, kind, N, A, 2000, hv)
    pcm = pcm_bytes(N, 2 * F, 24, 21)
    c0, c1 = np.ascontiguousarray(pcm[:, :F * 6]), np.ascontiguousarray(pcm[:, F * 6:])
    try:
        outputs_match(oracle, kind, eng, chains, packets, c0, npk, fpp, "before:")
        tx = eng.get_spdif_tx()
        pm = eng.get_preset_mute()
        assert (eng.set_rate_device(rates, inst0=inst0) == CURRENT).all()
        for k in range(n):
            i = inst0 + k
            chains[i] = switched(oracle, kind, chains[i], sts[i], packets[i:i + 1], hv[i], P0[i]["preset_mute_gain"], A, float(rates[k]))
        assert eng.get_spdif_tx().tobytes() == tx.tobytes() and eng.get_preset_mute().tobytes() == pm.tobytes()
        outputs_match(oracle, kind, eng, chains, packets, c1, npk, fpp, "after:")
    finally:
        eng.close()


# ---- 3. gains are not touched -------------------------------------------------------------------------------------------
def everything(eng, pcm, npk, fpp):
    blob = eng.state_export()
    collected = eng.collect_bulk_device()
    return [blob, *collected, *eng.process_host(pcm, 24, npk, fpp)]


@pytest.mark.parametrize("how", ["taylor", "exact", "preset"])
@pytest.mark.parametrize("kind", KINDS)
def test_gains_are_not_touched(kind, how):
    A, B = 96000.0, 192000.0                                   # upward: no band leaves the SVF; every recipe below 0.45 A
    npk, fpp = 2, 96
    if how == "preset":
        _, _, images, slots = fixture(kind)
        n = images.shape[0]
        configure = lambda e, fs: e.apply_preset_device(images, fs, slots=slots, host=hv)   # noqa: E731
    else:
        n = 21
        packets = packets_for(kind, n, 3000)
        configure = lambda e, fs: e.apply_bulk_device(packets, fs, host=hv, exact_db=how == "exact")   # noqa: E731
    hv = host_records(n, 31)
    pcm = pcm_bytes(n, npk * fpp, 24, 32)
    eng, twin = engine(kind, n, npk * fpp), engine(kind, n, npk * fpp)
    try:
        assert not configure(eng, A).any() and not configure(twin, B).any()
        assert (eng.set_rate_device(np.full(n, B, np.float32)) == CURRENT).all()
        for k, (x, y) in enumerate(zip(everything(eng, pcm, npk, fpp), everything(twin, pcm, npk, fpp))):
            assert np.ascontiguousarray(x).tobytes() == np.ascontiguousarray(y).tobytes(), f"item {k}"
    finally:
        eng.close()
        twin.close()


# ---- 4. clamps carry over -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_clamps_carry_over(libm, kind):
    oracle, q28 = libm, is_q(kind)
    n = 5
    packets = packets_for(kind, n, 4000)
    packets["eq"]["type"][:, :, 0] = 2                         # peaking at 30 kHz: inside 0.45 * 96 kHz, above 0.45 * 44.1 kHz
    packets["eq"]["freq"][:, :, 0] = 30000.0
    packets["eq"]["gain_db"][:, :, 0] = 6.0
    eng = engine(kind, n, 64)
    try:
        assert not eng.apply_bulk_device(packets, 96000.0).any()
        assert (eng.collect_bulk_device()[0]["eq"]["freq"][:, :roles(kind), 0] == np.float32(30000.0)).all()
        assert (eng.set_rate_device([44100.0] * n) == CURRENT).all()
        base = eng.download_biquads()
        assert (eng.set_rate_device([96000.0] * n) == CURRENT).all()
        got, (rec, _, _) = eng.download_biquads(), eng.collect_bulk_device()
        assert (rec["eq"]["freq"][:, :roles(kind), 0] == np.float32(44100.0) * np.float32(0.45)).all()
        for i in range(n):
            st = api.bulk_state_defaults(platform(kind))
            assert api.bulk_params_apply(rec[i:i + 1], st) == 0
            assert same_bits(got[i], policy_biquads(oracle, q28, st, base[i], 96000.0)), f"instance {i}"
    finally:
        eng.close()


# ---- 5. delays ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_delays(libm, kind):
    oracle, q28 = libm, is_q(kind)
    A, B = (16000.0, 32000.0) if q28 else (32000.0, 64000.0)
    MAX = 2048 if q28 else 4096
    n_out = roles(kind) - 2
    N, npk, fpp = 6, 3, 64
    assert api.delay_samples(0.008, 44100.0) == 0 and api.delay_samples(0.008, 192000.0) == 1
    assert api.delay_samples(64.0, B) == MAX and api.delay_samples(64.0, A) == MAX // 2
    rates = np.array([192000.0, B, B, B, B, B], np.float32)
    delays = np.zeros((N, n_out), np.float32)
    delays[0, 0] = 0.008                                       # 0 samples at 44.1 kHz, 1 at 192 kHz
    delays[1, 0] = 64.0                                        # exactly MAX at B: aliases to no delay
    delays[2, 1] = 64.0
    delays[4, -1] = 3.0                                        # row 3: the sub's SUB_ALIGN_SAMPLES term alone
    delays[5] = np.linspace(0.0, 40.0, n_out)
    packets = packets_for(kind, N, 5000, fmax=0.44 * A, versions=(6,))
    packets["outputs"]["delay_ms"][:, :n_out] = delays
    rates[0], A0 = 192000.0, 44100.0                           # instance 0 switches 44.1 -> 192 kHz
    hv = host_records(N, 51)
    P0 = initial(kind, N, A, 5100)[1]                          # preset-mute gain 1
    pcm = pcm_bytes(N, npk * fpp, 24, 52)
    eng, twin = engine(kind, N, npk * fpp), engine(kind, N, npk * fpp)
    try:
        for e in (eng, twin):
            e.set_params(P0)
        assert not eng.apply_bulk_device(packets[:1], A0, host=hv[:1]).any()
        assert not eng.apply_bulk_device(packets[1:], A, inst0=1, host=hv[1:]).any()
        for i in range(N):
            assert not twin.apply_bulk_device(packets[i:i + 1], float(rates[i]), inst0=i, host=hv[i:i + 1]).any()
        assert (eng.set_rate_device(rates) == CURRENT).all()
        ia, ib = eng.export_instances(), twin.export_instances()
        for i in range(N):
            assert ia[i].tobytes() == ib[i].tobytes(), f"instance {i}: image against an engine configured at {rates[i]} Hz"
        spdif, _, _ = eng.process_host(pcm, 24, npk, fpp)
        dly = []
        for i in range(N):
            st = api.bulk_state_defaults(platform(kind))
            rc, P = expected(oracle, st, packets[i:i + 1], float(rates[i]), hv[i], False)
            assert rc == 0
            P["preset_mute_gain"] = P0[i]["preset_mute_gain"]
            dly.append([int(o["delay_samples"]) for o in P[0]["matrix"]["outputs"][:n_out]])
            zero = np.zeros((roles(kind), L.MAX_BANDS), L.BIQUAD_Q28 if q28 else L.BIQUAD_F32)
            ch = (make_orc_chain_q28 if q28 else make_orc_chain)(oracle, P[0], policy_biquads(oracle, q28, st, zero, float(rates[i])))
            ws, _ = run_oracle(oracle, kind, ch, pcm[i], 24, npk, fpp)
            assert np.array_equal(spdif[i], ws), f"instance {i}: S/PDIF words"
        assert dly[0][0] == 1 and dly[1][0] == MAX and dly[2][1] == MAX
        assert dly[3][-1] == api.delay_samples(0.0, B, True) > 0 and dly[3][:-1] == [0] * (n_out - 1)
    finally:
        eng.close()
        twin.close()


# ---- 6. stale and unset instances are refused -----------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_stale_and_unset_instances_are_left_alone(kind):
    N, fs = 12, 48000.0
    _, P0, bq0 = initial(kind, N, fs, 6000)
    packets = packets_for(kind, N, 6100)
    eng = engine(kind, N, 64)
    try:
        assert not eng.apply_bulk_device(packets[:8], fs).any()                  # 0..7 current, 8..11 unset
        eng.set_params(P0[2:4], inst0=2)                                          # 2, 3 stale
        eng.upload_biquads(bq0[5:6], inst0=5)                                     # 5 stale
        eng.process_host(pcm_bytes(N, 64, 16, 61), 16, 1, 64)
        marks = [CURRENT, CURRENT, STALE, STALE, CURRENT, STALE, CURRENT, CURRENT, UNSET, UNSET, UNSET, UNSET]
        before = eng.export_instances()
        inst0, n = 1, 9
        res = eng.set_rate_device(np.full(n, 96000.0, np.float32), inst0=inst0)
        assert list(res) == marks[inst0:inst0 + n]
        after = eng.export_instances()
        for i in range(N):
            same = before[i].tobytes() == after[i].tobytes()
            assert same == (not (inst0 <= i < inst0 + n and marks[i] == CURRENT)), f"instance {i} (mark {marks[i]})"
    finally:
        eng.close()


# ---- 7. per-instance rates across the staging chunk -----------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_per_instance_rates_across_the_staging_chunk(libm, kind):
    oracle, q28 = libm, is_q(kind)
    N, inst0, n, A = 1200, 64, 1100, 48000.0
    assert inst0 + n > CHUNK
    cycle = np.array([44100.0, 48000.0, 88200.0, 96000.0, 192000.0], np.float32)
    rates = cycle[np.arange(n) % cycle.size]
    packets = np.concatenate([wire_packet(platform(kind), 7000 + i % 97, version=6) for i in range(N)])
    eng = engine(kind, N, 64)
    try:
        assert not eng.apply_bulk_device(packets, A).any()
        base = eng.download_biquads()
        rec = eng.collect_bulk_device()[0]
        assert (eng.set_rate_device(rates, inst0=inst0) == CURRENT).all()
        got = eng.download_biquads()
        for i in range(N):
            if not inst0 <= i < inst0 + n:
                assert same_bits(got[i], base[i]), f"instance {i} outside the range"
                continue
            st = api.bulk_state_defaults(platform(kind))
            assert api.bulk_params_apply(rec[i:i + 1], st) == 0
            assert same_bits(got[i], policy_biquads(oracle, q28, st, base[i], float(rates[i - inst0]))), f"instance {i}"
    finally:
        eng.close()


# ---- 8. the run-time specialised K1 after every master band flips ----------------------------------------------------------
@pytest.mark.parametrize("kind", ["f32f", "f32s"])
def test_specialised_k1_after_flips(libm, kind):
    oracle = libm
    N, npk, fpp, A, B = 512, 1, 96, 44100.0, 96000.0            # 1024 master rows: the threshold of the specialised K1
    hv = np.zeros(N, L.BULK_HOST)
    _, P0, bq0 = initial(kind, N, A, 8000)
    packets = packets_for(kind, N, 8100, versions=(6,))
    packets["global"]["bypass"] = 0
    eq = packets["eq"]
    eq["type"][:, :2] = 2                                      # every master band peaking at 8 kHz: TDF2 at 44.1 kHz, SVF at 96 kHz
    eq["freq"][:, :2] = 8000.0
    eq["q"][:, :2] = 0.9
    eq["gain_db"][:, :2] = np.float32(3.0)
    eng = engine(kind, N, npk * fpp)
    try:
        eng.set_params(P0)
        assert not eng.apply_bulk_device(packets, A, host=hv).any()
        base = eng.download_biquads()
        assert (base["use_svf"][:, :2] == 0).all()
        assert (eng.set_rate_device(np.full(N, B, np.float32)) == CURRENT).all()
        got = eng.download_biquads()
        assert (got["use_svf"][:, :2, :10] == 1).all()
        pcm = pcm_bytes(N, npk * fpp, 24, 81)
        spdif, _, _ = eng.process_host(pcm, 24, npk, fpp)
        for i in range(0, N, 7):
            st = api.bulk_state_defaults(platform(kind))
            rc, P = expected(oracle, st, packets[i:i + 1], B, hv[i], False)
            assert rc == 0
            P["preset_mute_gain"] = P0[i]["preset_mute_gain"]
            ch = make_orc_chain(oracle, P[0], policy_biquads(oracle, False, record_state(oracle, kind, st, A), base[i], B))
            ws, _ = run_oracle(oracle, kind, ch, pcm[i], 24, npk, fpp)
            assert np.array_equal(spdif[i], ws), f"instance {i}"
    finally:
        eng.close()


# ---- 9. ordering behind an asynchronous process call ----------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_ordered_behind_asynchronous_process_calls(kind):
    N, fs = 64, 96000.0
    cadence = [96, 96]
    F = sum(cadence)
    pairs = 2 if is_q(kind) else 4
    packets = packets_for(kind, N, 9000)
    a, t = engine(kind, N, F), engine(kind, N, F)
    try:
        pcm = torch.from_numpy(pcm_bytes(N, F, 24, 91)).cuda()
        outs = {e: (torch.zeros((N, pairs, F, 2), dtype=torch.int32, device="cuda"), torch.zeros((N, F, 8), dtype=torch.int32, device="cuda"))
                for e in (a, t)}
        for e in (a, t):
            assert not e.apply_bulk_device(packets, fs).any()
        torch.cuda.synchronize()
        for e in (a, t):
            e.process_packets_device(pcm.data_ptr(), 24, cadence, outs[e][0].data_ptr(), outs[e][1].data_ptr())
        assert (a.set_rate_device(np.full(N, 44100.0, np.float32)) == CURRENT).all()     # right behind the asynchronous call
        t.sync()
        assert (t.set_rate_device(np.full(N, 44100.0, np.float32)) == CURRENT).all()
        for e in (a, t):
            e.process_packets_device(pcm.data_ptr(), 24, cadence, outs[e][0].data_ptr(), outs[e][1].data_ptr())
        a.sync()
        t.sync()
        assert torch.equal(outs[a][0], outs[t][0]) and torch.equal(outs[a][1], outs[t][1])
        assert a.state_export().tobytes() == t.state_export().tobytes()
    finally:
        a.close()
        t.close()


# ---- 10. argument errors write nothing ------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_bad_arguments_write_nothing(kind):
    N, fs = 6, 48000.0
    packets = packets_for(kind, N, 10000)
    eng, twin = engine(kind, N, 64), engine(kind, N, 64)
    fn = getattr(api.lib(), eng._PRE + "_set_rate_device")
    rates, res = np.full(N, 96000.0, np.float32), np.full(N, 77, np.int32)
    rp, sp = rates.ctypes.data, res.ctypes.data
    try:
        for e in (eng, twin):
            assert not e.apply_bulk_device(packets, fs).any()
        assert fn(None, 0, N, rp, sp) == EINVAL
        assert fn(eng._h, 0, N, None, sp) == EINVAL
        for bad in (0.0, -48000.0, float("nan"), float("inf")):
            rates[-1] = bad                                    # the last rate: every rate is checked before the first write
            assert fn(eng._h, 0, N, rp, sp) == EINVAL
        rates[-1] = 96000.0
        assert fn(eng._h, 1, N, rp, sp) == ERANGE
        assert fn(eng._h, 0xFFFFFFFF, 2, rp, sp) == ERANGE
        assert fn(eng._h, 2, 0, rp, sp) == 0
        assert (res == 77).all()
        assert eng.export_instances().tobytes() == twin.export_instances().tobytes()
        assert fn(eng._h, 0, N, rp, None) == 0                 # results may be NULL
        assert (twin.set_rate_device(rates) == CURRENT).all()
        assert eng.export_instances().tobytes() == twin.export_instances().tobytes()
    finally:
        eng.close()
        twin.close()
