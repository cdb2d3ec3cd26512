"""GPU: dspi_chain(q)_collect_bulk_device - REQ_GET_ALL_PARAMS from the configuration record every chain instance keeps in
device memory (bulk_ingest.cuh).  The expected bytes come from pieces pinned to the reference elsewhere: a shadow
dspi_bulk_state per instance taken through dspi_bulk_params_apply on the host, the recipe clamps of the oracle's coefficient
generator, and dspi_bulk_params_collect on the host."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                          # noqa: E402
from tests.bulk_cases import dims, wire_packet                                    # noqa: E402
from tests.chain_cases import pcm_bytes                                           # noqa: E402
from tests.util import same_bits                                                  # noqa: E402

KINDS = ["f32f", "f32s", "q28"]
EINVAL, ERANGE = -22, -34
CURRENT, STALE, UNSET = L.BULK_CURRENT, L.BULK_STALE, L.BULK_UNSET
CHUNK = 1024                                                                      # bulk::kChunk


def is_q(kind):
    return kind == "q28"


def platform(kind):
    return L.PLATFORM_RP2040 if is_q(kind) else L.PLATFORM_RP2350


def engine(kind, n, frames=64):
    return api.ChainEngineQ28(n, max_frames=frames) if is_q(kind) else api.ChainEngine(kind, n, max_frames=frames)


def host_records(n, seed):
    hv = np.zeros(n, L.BULK_HOST)
    rng = np.random.default_rng(seed)
    hv["volume_8_8"] = rng.integers(-40 * 256, 1, n)
    hv["host_mute"] = rng.random(n) < 0.1
    hv["reserved"] = rng.integers(0, 256, n)
    return hv


def audible(w):
    w["outputs"][0]["enabled"][:] = 1
    w["outputs"][0]["mute"][:] = 0
    w["crosspoints"][0]["enabled"][:] = 1
    return w


def dirty(w, seed):
    """The same settings with everything a well-behaved sender leaves zero filled in: reserved bytes, rows past the shape's
    channel and output counts, the control-plane sections, flags that are non-zero but not 1."""
    rng = np.random.default_rng(seed)
    nc, no = dims(int(w["header"][0]["platform_id"]))
    flag = lambda size=None: rng.choice([0, 1, 2, 0x80, 0xFF], size)              # noqa: E731
    junk = lambda size=None: rng.integers(1, 256, size)                           # noqa: E731
    fjunk = lambda size=None: rng.uniform(-50, 50, size).astype(np.float32)       # noqa: E731
    h = w["header"][0]
    h["num_input_channels"], h["max_bands"], h["fw_version_major"], h["fw_version_minor"] = junk(), junk(), junk(), junk()
    h["reserved"] = rng.integers(1, 2 ** 32)
    g = w["global"][0]
    g["bypass"], g["loudness_enabled"], g["reserved"] = flag(), flag(), junk(2)
    x = w["crossfeed"][0]
    x["enabled"], x["itd_enabled"], x["reserved"], x["reserved2"] = flag(), flag(), junk(), rng.integers(1, 2 ** 32)
    w["legacy"][0]["mute"], w["legacy"][0]["reserved"] = flag(3), junk()
    w["delays"][0]["delay_ms"][nc:] = fjunk(L.WIRE_MAX_CHANNELS - nc)
    cp = w["crosspoints"][0]
    cp["enabled"][:], cp["phase_invert"][:], cp["reserved"][:] = flag((2, L.WIRE_MAX_OUTPUTS)), flag((2, L.WIRE_MAX_OUTPUTS)), junk((2, L.WIRE_MAX_OUTPUTS, 2))
    cp["gain_db"][:, no:] = fjunk((2, L.WIRE_MAX_OUTPUTS - no))
    o = w["outputs"][0]
    o["enabled"][:], o["mute"][:], o["reserved"][:] = flag(L.WIRE_MAX_OUTPUTS), flag(L.WIRE_MAX_OUTPUTS), junk((L.WIRE_MAX_OUTPUTS, 2))
    o["gain_db"][no:], o["delay_ms"][no:] = fjunk(L.WIRE_MAX_OUTPUTS - no), fjunk(L.WIRE_MAX_OUTPUTS - no)
    p = w["pins"][0]
    p["num_pin_outputs"], p["pins"], p["reserved"] = junk(), junk(5), junk(2)
    e = w["eq"][0]
    e["reserved"][:] = junk((L.WIRE_MAX_CHANNELS, L.MAX_BANDS, 3))
    for f in ("freq", "q", "gain_db"):
        e[f][nc:] = fjunk((L.WIRE_MAX_CHANNELS - nc, L.MAX_BANDS))
    e["type"][nc:] = junk((L.WIRE_MAX_CHANNELS - nc, L.MAX_BANDS))
    raw = w.view(np.uint8).reshape(-1)
    for name in ("channel_names", "i2s_config"):
        off = L.WIRE_BULK.fields[name][1]
        raw[off:off + L.WIRE_BULK.fields[name][0].itemsize] = junk(L.WIRE_BULK.fields[name][0].itemsize)
    lv = w["leveller"][0]
    lv["enabled"], lv["lookahead"], lv["reserved"] = flag(), flag(), junk()
    w["preamp"][0]["reserved"], w["master_volume"][0]["reserved"] = junk(8), junk(12)
    return w


def packets_for(kind, n, seed, versions=(2, 3, 4, 5, 6), dirty_every=3):
    out = []
    for i in range(n):
        w = wire_packet(platform(kind), seed + i, version=versions[i % len(versions)])
        out.append(dirty(w, seed + i) if dirty_every and i % dirty_every == 1 else w)
    return np.concatenate(out)


class Shadow:
    """What a host that mirrors every call would hold: one dspi_bulk_state and one host record per instance."""

    def __init__(self, oracle, kind, n):
        self.oracle, self.q28, self.roles = oracle, is_q(kind), 7 if is_q(kind) else 11
        self.st = [api.bulk_state_defaults(platform(kind)) for _ in range(n)]
        self.hv = np.zeros(n, L.BULK_HOST)

    def clamp(self, i, fs):
        """dsp_recalculate_all_filters(): the clamps dsp_compute_coefficients() writes back into filter_recipes[][]"""
        rec = np.ascontiguousarray(self.st[i][0]["recipes"][:self.roles]).copy()
        bq = np.zeros((self.roles, L.MAX_BANDS), L.BIQUAD_Q28 if self.q28 else L.BIQUAD_F32)
        self.oracle.eq_coeffs(self.q28, rec, bq, fs)
        self.st[i][0]["recipes"][:self.roles] = rec

    def apply(self, packets, hv, fs, inst0=0, exact=False):
        codes = []
        for k in range(packets.shape[0]):
            rc = api.bulk_params_apply(packets[k:k + 1], self.st[inst0 + k], exact)
            codes.append(rc)
            if rc == 0:
                self.hv[inst0 + k] = hv[k]
                self.clamp(inst0 + k, fs)
        return codes

    def collect(self, inst0=0, n=None):
        n = len(self.st) - inst0 if n is None else n
        return np.concatenate([api.bulk_params_collect(self.st[inst0 + k]) for k in range(n)])


def assert_packets(got, want, what=""):
    for i in range(want.shape[0]):
        if got[i].tobytes() != want[i].tobytes():
            diff = [name for name in L.WIRE_BULK.names if got[i][name].tobytes() != want[i][name].tobytes()]
            raise AssertionError(f"{what} instance {i}: sections {diff} differ")
    assert got.shape == want.shape


def running(kind, n, fs, frames, seed):
    """An engine in a running configuration through the host route (preset-mute gain 1, so packets give audible output)."""
    q28 = is_q(kind)
    Ps = np.zeros(n, L.CHAIN_PARAMS_Q28 if q28 else L.CHAIN_PARAMS_F32)
    bqs = np.zeros((n, 7 if q28 else 11, L.MAX_BANDS), L.BIQUAD_Q28 if q28 else L.BIQUAD_F32)
    for i in range(n):
        st = api.bulk_state_defaults(platform(kind))
        assert api.bulk_params_apply(audible(wire_packet(platform(kind), seed + i)), st) == 0
        P, bq = api.bulk_state_to_chain(st, fs, -6 * 256)
        Ps[i], bqs[i] = P[0], bq[0]
    eng = engine(kind, n, frames)
    eng.set_params(Ps)
    eng.upload_biquads(bqs)
    return eng, Ps, bqs


# ---- 1. round trip ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fs", [44100.0, 48000.0, 96000.0])
@pytest.mark.parametrize("kind", KINDS)
def test_round_trip_matches_host_apply_clamp_collect(oracle, kind, fs):
    n = 101                                                    # neither a multiple of 32 nor of the CTA's 4 instances
    eng, sh = engine(kind, n), Shadow(oracle, kind, n)
    try:
        for exact in (False, True):
            packets, hv = packets_for(kind, n, 1000 + 500 * exact), host_records(n, 11 + exact)
            assert not eng.apply_bulk_device(packets, fs, host=hv, exact_db=exact).any()
            assert sh.apply(packets, hv, fs, exact=exact) == [0] * n
            got, ghv, codes = eng.collect_bulk_device()
            assert_packets(got, sh.collect(), f"exact_db={exact}")
            assert (codes == CURRENT).all() and ghv.tobytes() == hv.tobytes()
            assert (got["header"]["format_version"] == 6).all() and (got["header"]["payload_length"] == L.WIRE_BULK.itemsize).all()
    finally:
        eng.close()


# ---- 2. history ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_version_3_after_version_6_keeps_what_the_firmware_keeps(oracle, kind):
    n, fs = 24, 48000.0
    first, second = packets_for(kind, n, 2000, versions=(6,)), packets_for(kind, n, 2100, versions=(3,))
    hv1, hv2 = host_records(n, 21), host_records(n, 22)
    eng, sh = engine(kind, n), Shadow(oracle, kind, n)
    try:
        for pk, hv in ((first, hv1), (second, hv2)):
            assert not eng.apply_bulk_device(pk, fs, host=hv).any()
            assert sh.apply(pk, hv, fs) == [0] * n
        got, ghv, codes = eng.collect_bulk_device()
        want = sh.collect()
        assert_packets(got, want)
        assert ghv.tobytes() == hv2.tobytes() and (codes == CURRENT).all()
        mv = first["master_volume"]["master_volume_db"]
        mv = np.clip(np.where(np.isfinite(mv), mv, np.float32(0.0)), -128.0, 0.0).astype(np.float32)
        assert got["master_volume"]["master_volume_db"].tobytes() == mv.tobytes(), "the version 6 master volume stays in force"
        for side in range(2):
            assert got["preamp"]["preamp_db"][:, side].tobytes() == second["global"]["preamp_gain_db"].tobytes(), "legacy preamp on both sides"
        lv = got["leveller"]
        assert not lv["enabled"].any() and (lv["lookahead"] == 1).all() and (lv["amount"] == 50.0).all() and (lv["max_gain_db"] == 15.0).all()
    finally:
        eng.close()


# ---- 3. rejected packets ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_rejected_packets_leave_their_records(oracle, kind):
    n, fs, p = 12, 96000.0, platform(kind)
    first, hv1 = packets_for(kind, n, 3000), host_records(n, 31)
    second, hv2 = packets_for(kind, n, 3100, versions=(6,)), host_records(n, 32)
    h = second["header"]
    h["format_version"][1], h["format_version"][2], h["platform_id"][4] = 1, 7, 1 - p
    h["num_channels"][5] += 1
    h["num_output_channels"][7] -= 1
    h["payload_length"][8], h["payload_length"][10] = L.WIRE_BULK.itemsize - 64 - 1, L.WIRE_BULK.itemsize + 1
    want_codes = [0, -1, -1, 0, -2, -3, 0, -3, -4, 0, -4, 0]
    eng, sh = engine(kind, n), Shadow(oracle, kind, n)
    try:
        assert not eng.apply_bulk_device(first[:9], fs, host=hv1[:9]).any()          # instances 9..11 stay unset
        sh.apply(first[:9], hv1[:9], fs)
        before = eng.collect_bulk_device()
        assert list(eng.apply_bulk_device(second, fs, host=hv2)) == want_codes
        assert sh.apply(second, hv2, fs) == want_codes
        got, ghv, codes = eng.collect_bulk_device()
        want = sh.collect()
        for i, rc in enumerate(want_codes):
            if rc:
                assert got[i].tobytes() == before[0][i].tobytes() and ghv[i] == before[1][i] and codes[i] == before[2][i], f"instance {i} (code {rc})"
                assert codes[i] == (CURRENT if i < 9 else UNSET)
            else:
                assert got[i].tobytes() == want[i].tobytes() and ghv[i] == hv2[i] and codes[i] == CURRENT, f"instance {i}"
        assert not got[10:11].view(np.uint8).any()
    finally:
        eng.close()


# ---- 4. clamps ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_recipes_come_back_clamped(oracle, kind):
    n, fs, roles = 10, 44100.0, 7 if is_q(kind) else 11
    packets, hv = packets_for(kind, n, 4000, versions=(6,), dirty_every=0), host_records(n, 41)
    e = packets["eq"]
    e["type"][:, :roles] = np.random.default_rng(42).integers(1, 6, (n, roles, L.MAX_BANDS))
    e["gain_db"][:, :roles] = 3.0
    e["q"][:, :roles, 0::4], e["q"][:, :roles, 1::4] = 0.01, 45.0
    e["freq"][:, :roles, 2::4], e["freq"][:, :roles, 3::4] = 2.0, 30000.0
    eng, sh = engine(kind, n), Shadow(oracle, kind, n)
    try:
        assert not eng.apply_bulk_device(packets, fs, host=hv).any()
        sh.apply(packets, hv, fs)
        got = eng.collect_bulk_device()[0]
        assert_packets(got, sh.collect(), "after apply_bulk_device:")
        g = got["eq"][:, :roles]
        assert g["q"].min() == np.float32(0.1) and g["q"].max() == np.float32(20.0)
        assert g["freq"].min() == np.float32(10.0) and g["freq"].max() == np.float32(fs) * np.float32(0.45)

        inst0, m, fs2 = 3, 4, 96000.0                          # new recipes for a sub-range, at another rate
        rec = np.zeros((m, roles, L.MAX_BANDS), L.EQ_PARAM)
        rng = np.random.default_rng(43)
        rec["type"], rec["gain_db"] = rng.integers(0, 6, rec.shape), rng.choice([0.0, -4.0, 6.0], rec.shape)
        rec["freq"], rec["Q"] = rng.choice([1.0, 500.0, 12000.0, 47000.0], rec.shape), rng.choice([0.02, 0.7, 33.0], rec.shape)
        rec["channel"], rec["band"] = np.arange(roles)[None, :, None], np.arange(L.MAX_BANDS)[None, None, :]
        back = eng.set_eq_params_device(rec, fs2, inst0=inst0)
        for k in range(m):
            sh.st[inst0 + k][0]["recipes"][:roles] = rec[k]
            sh.clamp(inst0 + k, fs2)
            assert same_bits(back[k], sh.st[inst0 + k][0]["recipes"][:roles])
        got2, _, codes = eng.collect_bulk_device()
        assert_packets(got2, sh.collect(), "after set_eq_params_device:")
        outside = [i for i in range(n) if not inst0 <= i < inst0 + m]
        assert got2[outside].tobytes() == got[outside].tobytes() and (codes == CURRENT).all()
    finally:
        eng.close()


# ---- 5. dynamics --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_set_dynamics_edits_its_fields_only(oracle, kind):
    n, fs, inst0, m = 9, 48000.0, 2, 5
    packets, hv = packets_for(kind, n, 5000), host_records(n, 51)
    cfg = np.zeros(m, L.DYNAMICS_CONFIG)
    rng = np.random.default_rng(52)
    cfg["xf_enabled"], cfg["xf_itd_enabled"], cfg["xf_preset"] = rng.choice([0, 1, 3], m), rng.choice([0, 1, 9], m), rng.integers(0, 4, m)
    cfg["xf_custom_fc"], cfg["xf_custom_feed_db"] = rng.uniform(400, 2500, m), rng.uniform(0, 16, m)
    cfg["lev_enabled"], cfg["lev_lookahead"], cfg["lev_speed"] = rng.choice([0, 1, 5], m), rng.choice([0, 1, 2], m), rng.integers(0, 3, m)
    cfg["lev_amount"], cfg["lev_max_gain_db"], cfg["lev_gate_threshold_db"] = rng.uniform(0, 100, m), rng.uniform(0, 35, m), rng.uniform(-96, 0, m)
    cfg["loudness_ref_spl"], cfg["loudness_intensity_pct"], cfg["loudness_enabled"] = rng.uniform(70, 95, m), rng.uniform(0, 150, m), rng.choice([0, 1, 4], m)
    cfg["host_mute"], cfg["volume_8_8"] = rng.integers(0, 2, m), rng.integers(-40 * 256, 1, m)
    eng, sh = engine(kind, n), Shadow(oracle, kind, n)
    try:
        assert not eng.apply_bulk_device(packets, fs, host=hv).any()
        sh.apply(packets, hv, fs)
        before = eng.collect_bulk_device()
        eng.set_dynamics_device(cfg, fs, inst0=inst0)
        for k in range(m):
            s, c = sh.st[inst0 + k][0], cfg[k]
            for f in ("enabled", "itd_enabled", "preset", "custom_fc", "custom_feed_db"):
                s["crossfeed"][f] = c["xf_" + f]
            for f in ("enabled", "amount", "speed", "max_gain_db", "lookahead", "gate_threshold_db"):
                s["leveller"][f] = c["lev_" + f]
            for f in ("loudness_enabled", "loudness_ref_spl", "loudness_intensity_pct"):
                s[f] = c[f]
            sh.hv[inst0 + k]["volume_8_8"], sh.hv[inst0 + k]["host_mute"] = c["volume_8_8"], c["host_mute"]
        got, ghv, codes = eng.collect_bulk_device()
        assert_packets(got, sh.collect())
        assert ghv.tobytes() == sh.hv.tobytes() and (codes == CURRENT).all()
        outside = [i for i in range(n) if not inst0 <= i < inst0 + m]
        assert got[outside].tobytes() == before[0][outside].tobytes() and ghv[outside].tobytes() == before[1][outside].tobytes()
        changed = {name for i in range(inst0, inst0 + m) for name in L.WIRE_BULK.names if got[i][name].tobytes() != before[0][i][name].tobytes()}
        assert changed == {"global", "crossfeed", "leveller"}
    finally:
        eng.close()


# ---- 6. marks -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_marks_unset_stale_current(oracle, kind):
    n, fs = 40, 48000.0
    eng, Ps, bqs = running(kind, n, fs, 64, 6000)               # set_params and upload_biquads on a fresh engine: still unset
    sh = Shadow(oracle, kind, n)
    try:
        got, ghv, codes = eng.collect_bulk_device()
        assert (codes == UNSET).all() and not got.view(np.uint8).any() and not ghv.view(np.uint8).any()
        packets, hv = packets_for(kind, 30, 6100), host_records(30, 61)
        assert not eng.apply_bulk_device(packets, fs, inst0=5, host=hv).any()
        sh.apply(packets, hv, fs, inst0=5)
        current = eng.collect_bulk_device()
        assert list(current[2]) == [UNSET] * 5 + [CURRENT] * 30 + [UNSET] * 5
        assert_packets(current[0][5:35], sh.collect(5, 30))
        eng.set_params(Ps[8:14], inst0=8)
        eng.upload_biquads(bqs[20:40], inst0=20)
        got, ghv, codes = eng.collect_bulk_device()
        assert list(codes) == [UNSET] * 5 + [CURRENT] * 3 + [STALE] * 6 + [CURRENT] * 6 + [STALE] * 15 + [UNSET] * 5
        assert got.tobytes() == current[0].tobytes() and ghv.tobytes() == current[1].tobytes(), "packet bytes unchanged"
        again, hv2 = packets_for(kind, 4, 6200), host_records(4, 62)
        assert not eng.apply_bulk_device(again, fs, inst0=10, host=hv2).any()
        sh.apply(again, hv2, fs, inst0=10)
        got, _, codes = eng.collect_bulk_device(inst0=8, n=8)
        assert list(codes) == [STALE] * 2 + [CURRENT] * 4 + [CURRENT] * 2
        assert_packets(got, sh.collect(8, 8))
        eng.reset_state()
        assert eng.collect_bulk_device(inst0=8, n=8)[0].tobytes() == got.tobytes(), "reset_state leaves the record alone"
    finally:
        eng.close()


# ---- 7. feed-back -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_collected_packet_reconfigures_a_twin_identically(kind):
    n, fs, npk, fpp = 16, 48000.0, 2, 64
    packets = np.concatenate([audible(wire_packet(platform(kind), 7000 + i)) for i in range(n)])
    hv = host_records(n, 71)
    pcm = pcm_bytes(n, npk * fpp, 24, 72)
    eng, twin = running(kind, n, fs, npk * fpp, 7100)[0], running(kind, n, fs, npk * fpp, 7100)[0]
    try:
        for e in (eng, twin):
            assert not e.apply_bulk_device(packets, fs, host=hv, exact_db=True).any()
        got, ghv, _ = eng.collect_bulk_device()
        assert not twin.apply_bulk_device(got, fs, host=ghv, exact_db=True).any()
        again = twin.collect_bulk_device()
        assert again[0].tobytes() == got.tobytes() and again[1].tobytes() == ghv.tobytes() and (again[2] == CURRENT).all()
        assert same_bits(twin.download_biquads(), eng.download_biquads())
        a, b = eng.process_host(pcm, 24, npk, fpp), twin.process_host(pcm, 24, npk, fpp)
        assert a[0].any() and all(np.array_equal(x, y) for x, y in zip(a, b))
    finally:
        eng.close()
        twin.close()


# ---- 8. read-only and ordering ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_collect_is_read_only_and_ordered_behind_process_calls(oracle, kind):
    n, fs, npk, fpp = 21, 96000.0, 3, 96
    F = npk * fpp
    packets = np.concatenate([audible(wire_packet(platform(kind), 8000 + i)) for i in range(n)])
    hv = host_records(n, 81)
    pcm = pcm_bytes(n, 3 * F, 24, 82)
    c = [np.ascontiguousarray(pcm[:, k * F * 6:(k + 1) * F * 6]) for k in range(3)]
    sh = Shadow(oracle, kind, n)
    sh.apply(packets, hv, fs)
    want = sh.collect()
    a, b = running(kind, n, fs, F, 8100)[0], running(kind, n, fs, F, 8100)[0]
    try:
        for e in (a, b):
            assert not e.apply_bulk_device(packets, fs, host=hv).any()
        ra, rb = a.process_host(c[0], 24, npk, fpp), b.process_host(c[0], 24, npk, fpp)
        assert_packets(a.collect_bulk_device()[0], want)
        outs = []
        d_pcm = torch.from_numpy(c[1]).cuda()
        for e in (a, b):
            o = (torch.zeros((n, e._PAIRS, F, 2), dtype=torch.int32, device="cuda"), torch.zeros((n, F, 8), dtype=torch.int32, device="cuda"),
                 torch.zeros(n * e._STATUS.itemsize, dtype=torch.uint8, device="cuda"))
            outs.append(o)
        torch.cuda.synchronize()
        a.process_device(d_pcm.data_ptr(), 24, npk, fpp, *(t.data_ptr() for t in outs[0]))
        assert_packets(a.collect_bulk_device()[0], want, "behind an asynchronous process call:")
        b.process_device(d_pcm.data_ptr(), 24, npk, fpp, *(t.data_ptr() for t in outs[1]))
        a.sync()
        b.sync()
        assert outs[0][0].any() and all(torch.equal(x, y) for x, y in zip(outs[0], outs[1]))
        sa, sb = a.process_subframes_host(c[2], 24, [fpp] * npk), b.process_subframes_host(c[2], 24, [fpp] * npk)
        for x, y in zip(ra + sa, rb + sb):
            assert np.array_equal(x, y)
        assert np.array_equal(a.state_export(), b.state_export())
    finally:
        a.close()
        b.close()


# ---- 9. limits ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_ranges_across_the_staging_chunk_and_refused_calls(oracle, kind):
    N, inst0, n, fs = 2 * CHUNK + 200, 1000, CHUNK + 77, 48000.0
    base = packets_for(kind, 16, 9000)
    pick = np.random.default_rng(91).integers(0, 16, n)
    packets, hv = np.ascontiguousarray(base[pick]), host_records(n, 92)
    packets["global"]["loudness_ref_spl"] = (70.0 + np.arange(n) * 0.01).astype(np.float32)   # every instance its own packet
    sh16 = Shadow(oracle, kind, 16)
    sh16.apply(base, hv[:16], fs)
    want = np.ascontiguousarray(sh16.collect()[pick])
    want["global"]["loudness_ref_spl"] = packets["global"]["loudness_ref_spl"]
    eng = engine(kind, N)
    fn = getattr(api.lib(), eng._PRE + "_collect_bulk_device")
    try:
        assert not eng.apply_bulk_device(packets, fs, inst0=inst0, host=hv).any()
        got, ghv, codes = eng.collect_bulk_device(inst0=inst0 - 3, n=n + 6)
        assert list(codes[:3]) + list(codes[-3:]) == [UNSET] * 6 and (codes[3:-3] == CURRENT).all()
        assert_packets(got[3:-3], want)
        assert ghv[3:-3].tobytes() == hv.tobytes() and not got[:3].view(np.uint8).any() and not got[-3:].view(np.uint8).any()

        pk, h2, res = np.full(4, 0x5A, np.uint8).repeat(L.WIRE_BULK.itemsize), np.full(4, 0x5A5A5A5A, np.uint32), np.full(4, 77, np.int32)
        args = (pk.ctypes.data_as(C.c_void_p), h2.ctypes.data_as(C.c_void_p), res.ctypes.data_as(C.c_void_p))
        assert fn(None, 0, 4, *args) == EINVAL
        assert fn(eng._h, 0, 4, None, args[1], args[2]) == EINVAL
        assert fn(eng._h, N - 3, 4, *args) == ERANGE
        assert fn(eng._h, 0xFFFFFFFF, 2, *args) == ERANGE
        assert fn(eng._h, 5, 0, *args) == 0
        assert (pk == 0x5A).all() and (h2 == 0x5A5A5A5A).all() and (res == 77).all()
        assert fn(eng._h, inst0, 4, args[0], None, None) == 0                         # host and results are optional
        assert pk.tobytes() == want[:4].tobytes() and (h2 == 0x5A5A5A5A).all() and (res == 77).all()
    finally:
        eng.close()


# ---- 10. preset route ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_collected_packet_gives_the_preset_image_of_the_host_state(oracle, kind):
    n, fs = 10, 48000.0
    packets, hv = packets_for(kind, n, 10000), host_records(n, 101)
    eng, sh = engine(kind, n), Shadow(oracle, kind, n)
    try:
        assert not eng.apply_bulk_device(packets, fs, host=hv, exact_db=True).any()
        sh.apply(packets, hv, fs, exact=True)
        got = eng.collect_bulk_device()[0]
        for i in range(n):
            st = api.bulk_state_defaults(platform(kind))
            assert api.bulk_params_apply(got[i:i + 1], st, True) == 0
            image, want = api.preset_slot_collect(st, i % 10), api.preset_slot_collect(sh.st[i], i % 10)
            assert image.size == api.preset_slot_size(platform(kind)) and np.array_equal(image, want), f"instance {i}"
    finally:
        eng.close()
