"""GPU: dspi_chain(q)_apply_bulk_device - WireBulkParams packets for many instances, from wire bytes to engine records on
the device (bulk_ingest.cuh).  The expected records come from the pinned pieces: dspi_bulk_params_apply on the host gives
the state (byte-identical to the reference's bulk_params.c); the oracle's generators under the libm policy give the derived
records; the two conversions that call powf (exact dB, master volume) are restated here in double, rounded once."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                          # noqa: E402
from tests.bulk_cases import wire_packet                                          # noqa: E402
from tests.chain_cases import pcm_bytes                                           # noqa: E402
from tests.orc import make_orc_chain, make_orc_chain_q28, orc_chain_run, orc_chain_run_q28   # noqa: E402
from tests.util import same_bits                                                  # noqa: E402

KINDS = ["f32f", "f32s", "q28"]
EINVAL, ERANGE = -22, -34


def is_q(kind):
    return kind == "q28"


def platform(kind):
    return L.PLATFORM_RP2040 if is_q(kind) else L.PLATFORM_RP2350


def engine(kind, n, frames):
    return api.ChainEngineQ28(n, max_frames=frames) if is_q(kind) else api.ChainEngine(kind, n, max_frames=frames)


def host_records(n, seed):
    hv = np.zeros(n, L.BULK_HOST)
    rng = np.random.default_rng(seed)
    hv["volume_8_8"] = rng.integers(-40 * 256, 1, n)
    hv["host_mute"] = rng.random(n) < 0.1
    return hv


def policy_linear(db):
    """10^(dB/20) evaluated in double, rounded once (DESIGN §6)."""
    return np.float32(10.0 ** float(np.float32(db) / np.float32(20.0)))


def expected(oracle, st, w, fs, hv, exact):
    """(code, chain params [1] or None): bulk_params_apply on ``st`` (in place), then what the main loop derives, under the
    libm policy.  The recipes to apply are st["recipes"]."""
    rc = api.bulk_params_apply(w, st, exact)
    if rc:
        return rc, None
    s = st[0]
    q28 = int(s["platform"]) == L.PLATFORM_RP2040
    f2i = oracle.lib.orc_f2i_sat
    if exact:
        for rec in (s["crosspoints"].reshape(-1), s["outputs"]):
            for r in rec:
                r["gain_linear"] = policy_linear(r["gain_db"])
        for i in range(2):
            s["preamp_linear"][i] = policy_linear(s["preamp_db"][i])
            s["preamp_q28"][i] = f2i(float(s["preamp_linear"][i] * np.float32(2 ** 28)))
    if int(w["header"][0]["format_version"]) >= 6:
        lin = np.float32(0.0) if s["master_volume_db"] <= -128.0 else policy_linear(s["master_volume_db"])
        s["master_volume_linear"] = lin
        s["master_volume_q15"] = f2i(float(lin * np.float32(32768.0)))
    P, _ = api.bulk_state_to_chain(st, fs, int(hv["volume_8_8"]), bool(hv["host_mute"]))
    base = P.ctypes.data
    off = {k: P.dtype.fields[k][1] for k in ("crossfeed", "leveller", "loudness")}
    xcfg = np.ascontiguousarray(s["crossfeed"]).reshape(1)
    (oracle.lib.orc_xfeed_coeffs_q28 if q28 else oracle.lib.orc_xfeed_coeffs_f32)(base + off["crossfeed"], xcfg.ctypes.data, fs)
    lcfg = np.ascontiguousarray(s["leveller"]).reshape(1)
    oracle.lib.orc_lev_coeffs_compute(base + off["leveller"], lcfg.ctypes.data, fs)
    tab = np.zeros((L.LOUD_STEPS, 2), L.LOUD_Q28 if q28 else L.LOUD_F32)
    (oracle.lib.orc_loud_table_q28 if q28 else oracle.lib.orc_loud_table_f32)(tab.ctypes.data, float(s["loudness_ref_spl"]),
                                                                              float(s["loudness_intensity_pct"]), fs)
    idx = C.c_uint8()
    assert oracle.lib.orc_host_vol_mul(int(hv["volume_8_8"]), C.byref(idx)) == int(P[0]["host_vol_mul"])
    P["loudness"][0] = tab[idx.value]
    n_out = 5 if q28 else 9
    for o in range(n_out):
        want = oracle.lib.orc_delay_samples(float(s["outputs"][o]["delay_ms"]), fs, int(o == n_out - 1), 2048 if q28 else 4096)
        assert int(P[0]["matrix"]["outputs"][o]["delay_samples"]) == want
    return 0, P


def policy_biquads(oracle, q28, st, base, fs):
    """dsp_recalculate_all_filters() on ``base`` [roles, 12] (coefficients replaced, state kept unless the topology flips)."""
    roles = base.shape[0]
    rec = np.ascontiguousarray(st[0]["recipes"][:roles]).copy()
    bq = np.ascontiguousarray(base).copy()
    oracle.eq_coeffs(q28, rec, bq, fs)
    return bq


def live_filters(chain, q28):
    roles = 7 if q28 else 11
    dt = L.BIQUAD_Q28 if q28 else L.BIQUAD_F32
    out = np.zeros((roles, L.MAX_BANDS), dt)
    for r in range(roles):
        C.memmove(out[r].ctypes.data, C.addressof(chain.filters[r]), L.MAX_BANDS * dt.itemsize)
    return out


def replace_records(oracle, old, P, st, fs, q28):
    """What the main loop does to a running instance after an accepted packet: new records and coefficients; running
    state kept, except the crossfeed's (crossfeed_compute_coefficients clears it)."""
    bq = policy_biquads(oracle, q28, st, live_filters(old, q28), fs)
    new = (make_orc_chain_q28 if q28 else make_orc_chain)(oracle, P[0], bq)
    for f in ("loud_state", "levs", "delay_lines", "delay_widx", "pdm", "peaks", "clip_flags"):
        setattr(new, f, getattr(old, f))
    return new


def initial(kind, n, fs, seed):
    """A running configuration through the host route: states, params, biquads."""
    q28 = is_q(kind)
    sts, Ps = [], np.zeros(n, L.CHAIN_PARAMS_Q28 if q28 else L.CHAIN_PARAMS_F32)
    bqs = np.zeros((n, 7 if q28 else 11, L.MAX_BANDS), L.BIQUAD_Q28 if q28 else L.BIQUAD_F32)
    for i in range(n):
        st = api.bulk_state_defaults(platform(kind))
        w = wire_packet(platform(kind), seed + i)
        w["outputs"][0]["enabled"][:] = 1
        w["outputs"][0]["mute"][:] = 0
        w["crosspoints"][0]["enabled"][:] = 1
        w["master_volume"][0]["master_volume_db"] = np.float32(-2.0 * (i % 3))
        assert api.bulk_params_apply(w, st) == 0
        P, bq = api.bulk_state_to_chain(st, fs, -6 * 256)
        Ps[i], bqs[i] = P[0], bq[0]
        sts.append(st)
    return sts, Ps, bqs


def audible(w):
    w["outputs"][0]["enabled"][:] = 1
    w["crosspoints"][0]["enabled"][:] = 1
    return w


def run_oracle(oracle, kind, chain, data, bit_depth, npk, fpp):
    if is_q(kind):
        return orc_chain_run_q28(oracle, chain, data, bit_depth, npk, fpp)
    return orc_chain_run(oracle, kind, chain, data, bit_depth, npk, fpp)


# ---- 1. coefficients, bit-exact --------------------------------------------------------------------------------------
@pytest.mark.parametrize("fs", [44100.0, 48000.0, 96000.0])
@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_coefficients_match_the_oracle_policy(oracle, kind, fs):
    n, q28 = 37, is_q(kind)                                   # neither a multiple of 32 nor of the CTA's 4 instances
    packets = np.concatenate([wire_packet(platform(kind), 1000 + i, version=2 + i % 5) for i in range(n)])
    eng = engine(kind, n, 96)
    oracle.set_libm_f64(1)
    try:
        base = eng.download_biquads()
        res = eng.apply_bulk_device(packets, fs, host=host_records(n, 5))
        got = eng.download_biquads()
        assert not res.any()
        for i in range(n):
            st = api.bulk_state_defaults(platform(kind))
            assert api.bulk_params_apply(packets[i:i + 1], st) == 0
            want = policy_biquads(oracle, q28, st, base[i], fs)
            assert same_bits(got[i], want), f"instance {i} (wire version {2 + i % 5})"
    finally:
        eng.close()
        oracle.set_libm_f64(0)


# ---- 2. end to end on a running engine --------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_running_engine_continues_like_the_main_loop(oracle, kind):
    q28 = is_q(kind)
    N, inst0, n, npk, fpp, fs = 13, 3, 7, 4, 96, 96000.0
    F = npk * fpp
    sts, P0, bq0 = initial(kind, N, fs, 2000)
    pcm = pcm_bytes(N, 2 * F, 24, 21)
    c0, c1 = np.ascontiguousarray(pcm[:, :F * 6]), np.ascontiguousarray(pcm[:, F * 6:])
    packets = np.concatenate([audible(wire_packet(platform(kind), 2100 + i, version=2 + i % 5)) for i in range(n)])
    hv = host_records(n, 22)
    sub_o = 4 if q28 else 8
    oracle.set_libm_f64(1)
    eng = engine(kind, N, F)
    try:
        eng.set_params(P0)
        eng.upload_biquads(bq0)
        chains = [(make_orc_chain_q28 if q28 else make_orc_chain)(oracle, P0[i], bq0[i]) for i in range(N)]
        eng.process_host(c0, 24, npk, fpp)
        for i in range(N):
            run_oracle(oracle, kind, chains[i], c0[i], 24, npk, fpp)
        res = eng.apply_bulk_device(packets, fs, inst0=inst0, host=hv)
        assert not res.any()
        enabled = {}
        for i in range(N):
            enabled[i] = bool(P0[i]["matrix"]["outputs"][sub_o]["enabled"])
        for k in range(n):
            rc, P = expected(oracle, sts[inst0 + k], packets[k:k + 1], fs, hv[k], False)
            assert rc == 0
            P["preset_mute_gain"] = P0[inst0 + k]["preset_mute_gain"]            # left alone by the call
            chains[inst0 + k] = replace_records(oracle, chains[inst0 + k], P, sts[inst0 + k], fs, q28)
            enabled[inst0 + k] = bool(P[0]["matrix"]["outputs"][sub_o]["enabled"])
        spdif, pdm, status = eng.process_host(c1, 24, npk, fpp)
        for i in range(N):
            ws, wp = run_oracle(oracle, kind, chains[i], c1[i], 24, npk, fpp)
            where = "inside" if inst0 <= i < inst0 + n else "outside"
            assert np.array_equal(spdif[i], ws), f"instance {i} ({where} the range): S/PDIF words"
            if enabled[i]:
                assert np.array_equal(pdm[i], wp), f"instance {i} ({where} the range): PDM bits"
            assert list(status[i]["peaks"]) == list(chains[i].peaks)[:len(status[i]["peaks"])], f"instance {i}: meters"
    finally:
        eng.close()
        oracle.set_libm_f64(0)


# ---- 3. rejection -------------------------------------------------------------------------------------------------------
def bad_packets(kind):
    p = platform(kind)
    out = [audible(wire_packet(p, 3000 + i)) for i in range(10)]
    out[1]["header"][0]["format_version"] = 1
    out[2]["header"][0]["format_version"] = 7
    out[3]["header"][0]["platform_id"] = 1 - p
    out[4]["header"][0]["num_channels"] += 1
    out[5]["header"][0]["num_output_channels"] -= 1
    out[6]["header"][0]["payload_length"] = L.WIRE_BULK.itemsize - 64 - 1
    out[7]["header"][0]["payload_length"] = L.WIRE_BULK.itemsize + 1
    return np.concatenate(out)


@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_rejected_packets_change_nothing(kind):
    N, npk, fpp, fs = 10, 3, 64, 48000.0
    F = npk * fpp
    _, P0, bq0 = initial(kind, N, fs, 3100)
    pcm = pcm_bytes(N, 2 * F, 16, 31)
    c0, c1 = np.ascontiguousarray(pcm[:, :F * 4]), np.ascontiguousarray(pcm[:, F * 4:])
    packets = bad_packets(kind)
    want = [api.bulk_params_apply(packets[i:i + 1], api.bulk_state_defaults(platform(kind))) for i in range(N)]
    assert want == [0, -1, -1, -2, -3, -3, -4, -4, 0, 0]
    freqs = np.geomspace(20.0, 20000.0, 16).astype(np.float32)
    eng, twin = engine(kind, N, F), engine(kind, N, F)
    try:
        for e in (eng, twin):
            e.set_params(P0)
            e.upload_biquads(bq0)
            e.process_host(c0, 16, npk, fpp)
        res = eng.apply_bulk_device(packets, fs)
        assert list(res) == want
        got_bq, twin_bq = eng.download_biquads(), twin.download_biquads()
        got_r, twin_r = eng.response(freqs, fs), twin.response(freqs, fs)
        got, ref = eng.process_host(c1, 16, npk, fpp), twin.process_host(c1, 16, npk, fpp)
        blob, twin_blob = eng.state_export(), twin.state_export()
        for i in range(N):
            same = same_bits(got_bq[i], twin_bq[i]) and np.array_equal(got_r[i].view(np.uint32), twin_r[i].view(np.uint32)) and \
                all(np.array_equal(a[i], b[i]) for a, b in zip(got[:2], ref[:2]))
            assert same == (want[i] != 0), f"instance {i} (code {want[i]})"
        assert blob.size == twin_blob.size and not np.array_equal(blob, twin_blob)
    finally:
        eng.close()
        twin.close()


# ---- 4. gains and guards ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_gains_and_master_volume_guards(oracle, kind, exact):
    q28 = is_q(kind)
    mvs = [np.nan, np.inf, -np.inf, -128.0, -200.0, 3.0, -6.0]
    N, npk, fpp, fs = len(mvs), 3, 64, 48000.0
    F = npk * fpp
    packets = np.concatenate([audible(wire_packet(platform(kind), 4000 + i)) for i in range(N)])
    for i in range(N):
        w = packets[i:i + 1]
        w["master_volume"]["master_volume_db"] = np.float32(mvs[i])
        w["outputs"]["mute"][:] = 0
        g = w["crosspoints"]["gain_db"]
        g[0, 0, :4] = [0.0, -60.0, -70.0, 25.0]                   # exactly 0 dB, the clamp edge, beyond both clamps
        w["outputs"]["gain_db"][0, :3] = [0.0, 20.0, -61.0]
        w["global"]["loudness_enabled"] = 0
    hv = np.zeros(N, L.BULK_HOST)
    pcm = pcm_bytes(N, F, 16, 41)
    freqs = np.geomspace(20.0, 20000.0, 24).astype(np.float32)
    oracle.set_libm_f64(1)
    eng, twin = engine(kind, N, F), engine(kind, N, F)
    try:
        base = eng.download_biquads()
        Ps = np.zeros(N, L.CHAIN_PARAMS_Q28 if q28 else L.CHAIN_PARAMS_F32)
        bqs = base.copy()
        sts = []
        for i in range(N):
            st = api.bulk_state_defaults(platform(kind))
            rc, P = expected(oracle, st, packets[i:i + 1], fs, hv[i], exact)
            assert rc == 0
            Ps[i], bqs[i] = P[0], policy_biquads(oracle, q28, st, base[i], fs)
            sts.append(st)
        assert [float(s[0]["master_volume_linear"]) for s in sts[:6]] == [1.0, 1.0, 1.0, 0.0, 0.0, 1.0]
        eng.set_params(initial(kind, N, fs, 4100)[1])             # another configuration (preset-mute gain 1: not the call's to set)
        twin.set_params(Ps)
        twin.upload_biquads(bqs)
        assert not eng.apply_bulk_device(packets, fs, host=hv, exact_db=exact).any()
        assert np.array_equal(eng.response(freqs, fs).view(np.uint32), twin.response(freqs, fs).view(np.uint32)), "parameter rows"
        spdif, pdm, status = eng.process_host(pcm, 16, npk, fpp)
        for i in range(N):
            ch = (make_orc_chain_q28 if q28 else make_orc_chain)(oracle, Ps[i], bqs[i])
            ws, _ = run_oracle(oracle, kind, ch, pcm[i], 16, npk, fpp)
            assert np.array_equal(spdif[i], ws), f"instance {i} (master volume {mvs[i]} dB)"
    finally:
        eng.close()
        twin.close()
        oracle.set_libm_f64(0)


# ---- 5. distance to the host route --------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_distance_to_the_host_route(kind):
    q28 = is_q(kind)
    N, npk, fpp, fs = 40, 2, 96, 96000.0
    F = npk * fpp
    packets = np.concatenate([audible(wire_packet(platform(kind), 5000 + i, version=5)) for i in range(N)])
    hv = host_records(N, 51)
    Ps = np.zeros(N, L.CHAIN_PARAMS_Q28 if q28 else L.CHAIN_PARAMS_F32)
    bqs = np.zeros((N, 7 if q28 else 11, L.MAX_BANDS), L.BIQUAD_Q28 if q28 else L.BIQUAD_F32)
    for i in range(N):
        st = api.bulk_state_defaults(platform(kind))
        assert api.bulk_params_apply(packets[i:i + 1], st) == 0
        P, bq = api.bulk_state_to_chain(st, fs, int(hv[i]["volume_8_8"]), bool(hv[i]["host_mute"]))
        Ps[i], bqs[i] = P[0], bq[0]
    eng, twin = engine(kind, N, F), engine(kind, N, F)
    try:
        Pinit = initial(kind, N, fs, 5100)[1]                     # another configuration; a v5 packet leaves its master volume in force
        Pinit["master_volume_q15" if q28 else "master_volume_linear"] = 32768 if q28 else 1.0
        eng.set_params(Pinit)
        twin.set_params(Ps)
        twin.upload_biquads(bqs)
        assert not eng.apply_bulk_device(packets, fs, host=hv).any()
        got, host = eng.download_biquads(), twin.download_biquads()
        if q28:
            for f in ("b0", "b1", "b2", "a1", "a2"):
                assert np.max(np.abs(got[f].astype(np.int64) - host[f].astype(np.int64))) <= 512, f
        else:
            for f in ("b0", "b1", "b2", "a1", "a2", "sva1", "sva2", "sva3", "svm0", "svm1", "svm2"):
                assert float(np.max(np.abs(got[f] - host[f]))) <= 1e-6, f
            for f in ("use_svf", "svf_type"):
                assert np.array_equal(got[f], host[f]), f
        assert np.array_equal(got["bypass"], host["bypass"])
        # gains and delays are made without libm: with flat EQs and the dynamics stages off the two routes render the same words
        flat = packets.copy()
        flat["eq"]["type"] = 0
        flat["global"]["loudness_enabled"] = 0
        flat["crossfeed"]["enabled"] = 0
        flat["leveller"]["enabled"] = 0
        for i in range(N):
            st = api.bulk_state_defaults(platform(kind))
            assert api.bulk_params_apply(flat[i:i + 1], st) == 0
            P, bq = api.bulk_state_to_chain(st, fs, int(hv[i]["volume_8_8"]), bool(hv[i]["host_mute"]))
            Ps[i], bqs[i] = P[0], bq[0]
        twin.set_params(Ps)
        twin.upload_biquads(bqs)
        assert not eng.apply_bulk_device(flat, fs, host=hv).any()
        pcm = pcm_bytes(N, F, 24, 52)
        a, b = eng.process_host(pcm, 24, npk, fpp), twin.process_host(pcm, 24, npk, fpp)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    finally:
        eng.close()
        twin.close()


# ---- 6. arguments -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_bad_arguments_write_nothing(kind):
    N, fs = 6, 48000.0
    _, P0, bq0 = initial(kind, N, fs, 6000)
    packets = np.concatenate([wire_packet(platform(kind), 6100 + i) for i in range(N)])
    hv, res = np.zeros(N, L.BULK_HOST), np.full(N, 77, np.int32)
    eng, twin = engine(kind, N, 64), engine(kind, N, 64)
    fn = getattr(api.lib(), eng._PRE + "_apply_bulk_device")
    pk, hp, rp = packets.ctypes.data, hv.ctypes.data, res.ctypes.data
    try:
        for e in (eng, twin):
            e.set_params(P0)
            e.upload_biquads(bq0)
        assert fn(None, 0, N, pk, hp, 0, C.c_float(fs), rp) == EINVAL
        assert fn(eng._h, 0, N, None, hp, 0, C.c_float(fs), rp) == EINVAL
        assert fn(eng._h, 0, N, pk, None, 0, C.c_float(fs), rp) == EINVAL
        assert fn(eng._h, 0, N, pk, hp, 0, C.c_float(fs), None) == EINVAL
        for bad in (0.0, -48000.0, float("nan"), float("inf")):
            assert fn(eng._h, 0, N, pk, hp, 0, C.c_float(bad), rp) == EINVAL
        assert fn(eng._h, 1, N, pk, hp, 0, C.c_float(fs), rp) == ERANGE
        assert fn(eng._h, 0xFFFFFFFF, 2, pk, hp, 0, C.c_float(fs), rp) == ERANGE
        assert fn(eng._h, 2, 0, pk, hp, 0, C.c_float(fs), rp) == 0
        assert (res == 77).all()
        assert same_bits(eng.download_biquads(), twin.download_biquads())
        pcm = pcm_bytes(N, 64, 16, 61)
        a, b = eng.process_host(pcm, 16, 1, 64), twin.process_host(pcm, 16, 1, 64)
        assert all(np.array_equal(x, y) for x, y in zip(a[:2], b[:2]))
        assert np.array_equal(eng.state_export(), twin.state_export())
    finally:
        eng.close()
        twin.close()
