"""GPU: dspi_chain(q)_edit_bulk_device - single fields of many instances' configuration edited on the device
(bulk_ingest.cuh edit_kernel), against the host route it is defined by: collect_bulk_device, the edits written over the
packets and host records in list order, apply_bulk_device at the same rate and gain conversion.  Running engines are
checked against oracle chains whose records were replaced under the call's state rules."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                          # noqa: E402
from tests.chain_cases import pcm_bytes                                           # noqa: E402
from tests.orc import make_orc_chain, make_orc_chain_q28                           # noqa: E402
from tests.test_bulk_device_gpu import engine, expected, host_records, initial, is_q, platform, policy_biquads, replace_records, run_oracle   # noqa: E402
from tests.test_preset_device_gpu import fixture                                  # noqa: E402
from tests.test_rate_switch_gpu import packets_for, roles                         # noqa: E402

CASES = [("f32f", 1), ("f32s", 1), ("f32s", 2), ("q28", 1)]                       # (kind, DSPI_F32_CPL: K1 geometry)
KINDS = ["f32f", "f32s", "q28"]
EINVAL, ERANGE = -22, -34
CURRENT, STALE, UNSET = L.BULK_CURRENT, L.BULK_STALE, L.BULK_UNSET
EDIT_CHUNK = 65536                                                                 # bulk::kEditChunk


@pytest.fixture
def libm(oracle):
    oracle.set_libm_f64(1)
    yield oracle
    oracle.set_libm_f64(0)


def outs(kind):
    return roles(kind) - 2


def random_field(rng, kind):
    """(path, value) of one editable field or section, with values a console could send"""
    u = lambda a, b: np.float32(rng.uniform(a, b))                                # noqa: E731
    bit = lambda p: int(rng.random() < p)                                         # noqa: E731
    side, ch, b = int(rng.integers(2)), int(rng.integers(roles(kind))), int(rng.integers(12))
    o = int(rng.integers(min(outs(kind) + (rng.random() < 0.1), L.WIRE_MAX_OUTPUTS)))        # now and then a row past the shape
    if rng.random() < 0.05:
        ch = int(rng.integers(roles(kind), L.WIRE_MAX_CHANNELS)) if roles(kind) < L.WIRE_MAX_CHANNELS else ch   # rows past the shape
    c = int(rng.integers(18))
    if c == 0:
        return ("crosspoints", side, o), (bit(0.8), bit(0.2), (0, 0), u(-30, 6))
    if c == 1:
        return ("crosspoints", side, o, "gain_db"), u(-40, 10)
    if c == 2:
        return ("outputs", o, "enabled"), bit(0.8)
    if c == 3:
        return ("outputs", o, "mute"), bit(0.2)
    if c == 4:
        return ("outputs", o, "gain_db"), u(-20, 6)
    if c == 5:
        return ("outputs", o, "delay_ms"), u(0, 30) if rng.random() < 0.7 else np.float32(0)
    if c == 6:
        return ("outputs", o), (bit(0.8), bit(0.2), (0, 0), u(-20, 6), u(0, 10))
    if c == 7:
        return ("preamp", "preamp_db", side), u(-12, 6)
    if c == 8:
        return ("master_volume", "master_volume_db"), [u(-60, 0), np.float32(3.0), np.float32(-200.0)][int(rng.integers(3))]
    if c == 9:
        return ("global", "bypass"), bit(0.3)
    if c == 10:
        k = int(rng.integers(3))
        return [("global", "loudness_enabled"), ("global", "loudness_ref_spl"), ("global", "loudness_intensity_pct")][k], \
            [bit(0.5), u(70, 90), u(0, 100)][k]
    if c == 11:
        return ("crossfeed",), (bit(0.7), int(rng.integers(4)), bit(0.5), 0, u(300, 1500), u(-12, -2), 0)
    if c == 12:
        return ("leveller",), (bit(0.6), int(rng.integers(3)), bit(0.5), 0, u(0, 100), u(0, 20), u(-90, -40))
    if c in (13, 14):
        return ("eq", ch, b), (int(rng.integers(6)), (0, 0, 0), np.float32(20.0 * 1000.0 ** rng.random()), u(0.3, 8), u(-15, 15))
    if c == 15:
        return ("eq", ch, b, ["freq", "gain_db", "q"][int(rng.integers(3))] if rng.random() < 0.7 else "type"), None
    if c == 16:
        return [("legacy", "gain_db", int(rng.integers(3))), ("legacy", "mute", int(rng.integers(3))),
                ("delays", "delay_ms", int(rng.integers(2)))][int(rng.integers(3))], None
    return [("host", "volume_8_8"), ("host", "host_mute"), ("host",)][int(rng.integers(3))], None


def value_for(rng, path, value):
    if value is not None:
        return value
    name = path[-1] if isinstance(path[-1], str) else path[-2]
    if path == ("host",):
        return (int(rng.integers(-60 * 256, 1)), int(rng.random() < 0.2), 0)
    return {"freq": np.float32(20.0 * 1000.0 ** rng.random()), "gain_db": np.float32(rng.uniform(-15, 15)), "q": np.float32(rng.uniform(0.3, 8)),
            "type": int(rng.integers(6)), "mute": int(rng.random() < 0.5), "delay_ms": np.float32(rng.uniform(0, 5)),
            "volume_8_8": int(rng.integers(-60 * 256, 1)), "host_mute": int(rng.random() < 0.3)}[name]


def random_edits(rng, kind, insts, count):
    """BULK_EDIT [count] for the given instances, interleaved; about one in six rewrites a slice of a field another value of
    it wrote, so bytes overlap"""
    out = []
    while len(out) < count:
        path, value = random_field(rng, kind)
        e = L.bulk_edit(int(rng.choice(insts)), path, value_for(rng, path, value))
        n = int(e["length"][0])
        if n > 1 and rng.random() < 0.17:
            a = int(rng.integers(0, n - 1))
            z = int(rng.integers(a + 1, n + 1))
            part = np.zeros(1, L.BULK_EDIT)
            part["instance"], part["offset"], part["length"] = e["instance"], int(e["offset"][0]) + a, z - a
            part["bytes"][0, :z - a] = e["bytes"][0, a:z]
            e = part
        out.append(e)
    return np.concatenate(out)


def patched(P, H, edits):
    """the edits written over the collected packets and host records in list order"""
    n = P.shape[0]
    buf = np.concatenate([np.ascontiguousarray(P).view(np.uint8).reshape(n, 2896), np.ascontiguousarray(H).view(np.uint8).reshape(n, 4)], axis=1)
    for e in edits:
        o, k = int(e["offset"]), int(e["length"])
        buf[int(e["instance"]), o:o + k] = e["bytes"][:k]
    return np.ascontiguousarray(buf[:, :2896]).view(L.WIRE_BULK).reshape(n), np.ascontiguousarray(buf[:, 2896:]).view(L.BULK_HOST).reshape(n)


def host_route(twin, edits, fs, exact):
    P, H, marks = twin.collect_bulk_device()
    assert (marks == CURRENT).all()
    P2, H2 = patched(P, H, edits)
    assert not twin.apply_bulk_device(P2, fs, host=H2, exact_db=exact).any()


def everything(eng, pcm, npk, fpp):
    return [*eng.collect_bulk_device(), eng.export_instances(), *eng.process_host(pcm, 24, npk, fpp), eng.state_export()]


def assert_same(a, b):
    for k, (x, y) in enumerate(zip(a, b)):
        assert np.ascontiguousarray(x).tobytes() == np.ascontiguousarray(y).tobytes(), f"item {k}"


def configured(oracle, kind, n, fs, seed, hv):
    """An engine of n instances configured by version-6 packets (so every derived row, the master volume included, follows
    the record) on top of a host-route configuration with its preset-mute gains, and its oracle chains:
    (engine, packets, preset-mute gains, chains)."""
    q28 = is_q(kind)
    sts, P0, bq0 = initial(kind, n, fs, seed)
    packets = packets_for(kind, n, seed + 500, versions=(6,))
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
    return eng, packets, P0["preset_mute_gain"], chains


def pair(kind, n, frames):
    return engine(kind, n, frames), engine(kind, n, frames)


# ---- 1. equivalence with the host route ----------------------------------------------------------------------------------
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("kind,cpl", CASES)
def test_equals_the_host_route(monkeypatch, kind, cpl, exact):
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    N, fs, npk, fpp = 70, 96000.0, 2, 48
    rng = np.random.default_rng(100 + cpl + 10 * exact)
    packets, hv = packets_for(kind, N, 1100, versions=(6,)), host_records(N, 12)
    edits = random_edits(rng, kind, rng.choice(N, 23, replace=False), 600)
    eng, twin = pair(kind, N, npk * fpp)
    try:
        for e in (eng, twin):
            assert not e.apply_bulk_device(packets, fs, host=hv, exact_db=exact).any()
        res = eng.edit_bulk_device(edits, fs, exact_db=exact)
        assert res.shape == (len(edits),) and (res == CURRENT).all()
        host_route(twin, edits, fs, exact)
        pcm = pcm_bytes(N, npk * fpp, 24, 13)
        assert_same(everything(eng, pcm, npk, fpp), everything(twin, pcm, npk, fpp))
    finally:
        eng.close()
        twin.close()


# ---- 2. a running engine continues like oracle chains with replaced records ------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_running_engine_continues_like_the_oracle(libm, kind):
    oracle, q28 = libm, is_q(kind)
    N, npk, fpp, fs = 9, 2, 96, 96000.0
    F = npk * fpp
    hv = host_records(N, 23)
    hv["host_mute"] = 0
    eng, packets, pmg, chains = configured(oracle, kind, N, fs, 2300, hv)
    pcm = pcm_bytes(N, 2 * F, 24, 24)
    c0, c1 = np.ascontiguousarray(pcm[:, :F * 6]), np.ascontiguousarray(pcm[:, F * 6:])
    edits = np.concatenate([
        L.bulk_edit(0, ("crossfeed", "enabled"), 1), L.bulk_edit(1, ("crossfeed", "enabled"), 1),   # crossfeed on for the next call
    ])
    later = np.concatenate([
        L.bulk_edit(0, ("host", "volume_8_8"), -9 * 256),                          # crossfeed state kept
        L.bulk_edit(1, ("outputs", 0, "gain_db"), np.float32(-4.5)),               # crossfeed state kept
        L.bulk_edit(2, ("crossfeed", "custom_fc"), np.float32(650.0)),              # crossfeed state cleared
        L.bulk_edit(2, ("crossfeed", "preset"), 3),
        L.bulk_edit(3, ("eq", 2, 3), (L.PEAKING, (0, 0, 0), 2500.0, 1.2, 4.0)),
        L.bulk_edit(4, ("master_volume", "master_volume_db"), np.float32(-7.0)),
        L.bulk_edit(4, ("outputs", 1, "mute"), 1),
        L.bulk_edit(5, ("outputs", 0, "delay_ms"), np.float32(1.5)),
        L.bulk_edit(6, ("leveller",), (1, 1, 1, 0, 60.0, 12.0, -70.0)),
        L.bulk_edit(7, ("global", "loudness_ref_spl"), np.float32(80.0)),
    ])
    try:
        P, H, _ = eng.collect_bulk_device()
        for round_, (ed, chunk) in enumerate(((edits, c0), (later, c1))):
            assert (eng.edit_bulk_device(ed, fs) == CURRENT).all()
            P2, H2 = patched(P, H, ed)
            xf = {int(e["instance"]) for e in ed if L.edit_field(("crossfeed",))[0] <= int(e["offset"]) < L.edit_field(("crossfeed",))[0] + 16}
            for i in {int(e["instance"]) for e in ed}:
                st = api.bulk_state_defaults(platform(kind))
                rc, Pi = expected(oracle, st, P2[i:i + 1], fs, H2[i], False)
                assert rc == 0
                Pi["preset_mute_gain"] = pmg[i]
                new = replace_records(oracle, chains[i], Pi, st, fs, q28)
                if i not in xf:
                    for f in ("lp_state_L", "lp_state_R", "ap_state_L", "ap_state_R"):
                        setattr(new.xfeed, f, getattr(chains[i].xfeed, f))
                chains[i] = new
            P, H = P2, H2
            spdif, pdm, status = eng.process_host(chunk, 24, npk, fpp)
            for i, ch in enumerate(chains):
                ws, wp = run_oracle(oracle, kind, ch, chunk[i], 24, npk, fpp)
                assert np.array_equal(spdif[i], ws), f"round {round_} instance {i}: S/PDIF words"
                if P[i]["outputs"]["enabled"][roles(kind) - 3]:
                    assert np.array_equal(pdm[i], wp), f"round {round_} instance {i}: PDM bits"
    finally:
        eng.close()


# ---- 3. sparsity ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_instances_not_named_are_untouched(monkeypatch, kind, cpl):
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    N, fs = 200, 48000.0
    rng = np.random.default_rng(300 + cpl)
    named = [31, 32, 64, 97, 199]                                                 # mid-group, group starts, the engine's end
    eng = engine(kind, N, 64)
    try:
        assert not eng.apply_bulk_device(packets_for(kind, N, 3100), fs).any()
        eng.process_host(pcm_bytes(N, 64, 16, 31), 16, 1, 64)
        before = eng.export_instances()
        assert (eng.edit_bulk_device(random_edits(rng, kind, named, 300), fs) == CURRENT).all()
        after = eng.export_instances()
        for i in range(N):
            assert (before[i].tobytes() == after[i].tobytes()) == (i not in named), f"instance {i}"
    finally:
        eng.close()


@pytest.mark.parametrize("kind", KINDS)
def test_crosspoint_edit_at_another_rate_rederives_nothing_else(kind):
    N, A, B = 12, 96000.0, 44100.0
    packets = packets_for(kind, N, 3200)
    edits = np.concatenate([L.bulk_edit(i, ("crosspoints", i % 2, i % outs(kind), "gain_db"), np.float32(-2.5 - i)) for i in range(N)])
    eng, twin = pair(kind, N, 64)
    try:
        for e in (eng, twin):
            assert not e.apply_bulk_device(packets, A).any()
        bq, img = eng.download_biquads(), eng.export_instances().tobytes()
        assert (eng.edit_bulk_device(edits, B) == CURRENT).all()                  # at B: nothing rate-dependent moves
        assert (twin.edit_bulk_device(edits, A) == CURRENT).all()
        assert eng.download_biquads().tobytes() == bq.tobytes()
        assert eng.export_instances().tobytes() == twin.export_instances().tobytes() != img
    finally:
        eng.close()
        twin.close()


@pytest.mark.parametrize("kind", KINDS)
def test_preset_loaded_gains_are_kept(kind):
    fs, npk, fpp = 48000.0, 2, 64
    _, _, images, slots = fixture(kind)
    n = images.shape[0]
    hv = host_records(n, 33)
    eng, ref = pair(kind, n, npk * fpp)
    route = engine(kind, n, npk * fpp)
    try:
        for e in (eng, ref, route):
            assert not e.apply_preset_device(images, fs, slots=slots, host=hv).any()
        # host volume and mute written again with the values they have: the output gain rows are recomputed from the
        # linear gains the preset load made (flash conversion), so nothing changes
        edits = np.concatenate([L.bulk_edit(i, ("host",), hv[i].tobytes()) for i in range(n)])
        assert (eng.edit_bulk_device(edits, fs) == CURRENT).all()
        assert eng.export_instances().tobytes() == ref.export_instances().tobytes()
        host_route(route, edits, fs, False)                                       # the whole-instance route converts every gain again
        assert route.export_instances().tobytes() != ref.export_instances().tobytes()
        pcm = pcm_bytes(n, npk * fpp, 24, 34)
        assert_same(everything(eng, pcm, npk, fpp), everything(ref, pcm, npk, fpp))
    finally:
        eng.close()
        ref.close()
        route.close()


# ---- 4. stale and unset instances -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_stale_and_unset_instances_report_their_marks(kind):
    N, fs = 12, 48000.0
    _, P0, bq0 = initial(kind, N, fs, 4000)
    eng = engine(kind, N, 64)
    rng = np.random.default_rng(41)
    try:
        assert not eng.apply_bulk_device(packets_for(kind, 8, 4100), fs).any()    # 0..7 current, 8..11 unset
        eng.set_params(P0[2:4], inst0=2)                                          # 2, 3 stale
        eng.upload_biquads(bq0[5:6], inst0=5)                                     # 5 stale
        marks = [CURRENT, CURRENT, STALE, STALE, CURRENT, STALE, CURRENT, CURRENT, UNSET, UNSET, UNSET, UNSET]
        before = eng.export_instances()
        collected = eng.collect_bulk_device()
        edits = random_edits(rng, kind, np.arange(N), 200)
        res = eng.edit_bulk_device(edits, fs)
        assert list(res) == [marks[int(i)] for i in edits["instance"]]
        after = eng.export_instances()
        again = eng.collect_bulk_device()
        for i in range(N):
            assert (before[i].tobytes() == after[i].tobytes()) == (marks[i] != CURRENT), f"instance {i} (mark {marks[i]})"
            if marks[i] != CURRENT:
                assert again[0][i].tobytes() == collected[0][i].tobytes() and again[1][i].tobytes() == collected[1][i].tobytes()
        assert list(again[2]) == marks
    finally:
        eng.close()


# ---- 5. order: last write wins, across the staging chunks ----------------------------------------------------------------
@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_list_order_across_the_staging_chunks(kind):
    N, fs = 1100, 48000.0                                                          # more distinct instances than one chunk holds
    rng = np.random.default_rng(51)
    packets = packets_for(kind, N, 5100, versions=(6,))
    fill = np.repeat(L.bulk_edit(7, ("outputs", 1, "gain_db"), np.float32(0.0)), EDIT_CHUNK + 1)
    fill["bytes"][:, :4] = np.linspace(-1.0, -20.0, EDIT_CHUNK + 1, dtype=np.float32)[:, None].view(np.uint8)
    # one instance fills the first chunk and goes on into the next one; then more distinct instances than a chunk holds
    edits = np.concatenate([fill, random_edits(rng, kind, np.arange(N), 2500)])
    eng, twin = pair(kind, N, 64)
    try:
        for e in (eng, twin):
            assert not e.apply_bulk_device(packets, fs).any()
        assert (eng.edit_bulk_device(edits, fs) == CURRENT).all()
        host_route(twin, edits, fs, False)
        for x, y in zip(eng.collect_bulk_device(), twin.collect_bulk_device()):
            assert x.tobytes() == y.tobytes()
        assert eng.export_instances().tobytes() == twin.export_instances().tobytes()
    finally:
        eng.close()
        twin.close()


# ---- 6. topology flips of every master band, bypass and mute edits ---------------------------------------------------------
@pytest.mark.parametrize("kind", ["f32f", "f32s"])
def test_specialised_k1_after_flips_and_skip_edits(libm, kind):
    oracle = libm
    N, npk, fpp, fs = 512, 1, 96, 96000.0                                          # 1024 master rows: the threshold of the specialised K1
    hv = np.zeros(N, L.BULK_HOST)
    _, P0, _ = initial(kind, N, fs, 6000)
    packets = packets_for(kind, N, 6100, versions=(6,))
    packets["global"]["bypass"] = 0
    eq = packets["eq"]
    eq["type"][:, :2] = L.PEAKING                                                  # every master band at 8 kHz: SVF at 96 kHz
    eq["freq"][:, :2] = 8000.0
    eq["q"][:, :2] = 0.9
    eq["gain_db"][:, :2] = np.float32(3.0)
    eng = engine(kind, N, npk * fpp)
    try:
        eng.set_params(P0)
        assert not eng.apply_bulk_device(packets, fs, host=hv).any()
        base = eng.download_biquads()
        assert (base["use_svf"][:, :2, :10] == 1).all()
        flips = np.concatenate([L.bulk_edit(i, ("eq", ch, b, "freq"), np.float32(14000.0)) for i in range(N) for ch in range(2) for b in range(12)])
        skips = np.concatenate([L.bulk_edit(i, ("global", "bypass"), 1) for i in range(0, N, 5)] +
                               [L.bulk_edit(i, ("outputs", 0, "mute"), 1) for i in range(1, N, 5)] +
                               [L.bulk_edit(i, ("outputs", 0, "enabled"), 0) for i in range(2, N, 5)])
        edits = np.concatenate([flips, skips])
        assert (eng.edit_bulk_device(edits, fs) == CURRENT).all()
        got = eng.download_biquads()
        assert (got["use_svf"][:, :2, :10] == 0).all()                              # 14 kHz: TDF2 above fs / 7.5
        P, H, _ = eng.collect_bulk_device()
        pcm = pcm_bytes(N, npk * fpp, 24, 61)
        spdif, _, _ = eng.process_host(pcm, 24, npk, fpp)
        for i in list(range(0, N, 7)) + [0, 1, 2, 5, 6, 7]:
            st = api.bulk_state_defaults(platform(kind))
            rc, Pi = expected(oracle, st, P[i:i + 1], fs, H[i], False)
            assert rc == 0
            Pi["preset_mute_gain"] = P0[i]["preset_mute_gain"]
            ch = make_orc_chain(oracle, Pi[0], policy_biquads(oracle, False, st, base[i], fs))
            ws, _ = run_oracle(oracle, kind, ch, pcm[i], 24, npk, fpp)
            assert np.array_equal(spdif[i], ws), f"instance {i}"
    finally:
        eng.close()


# ---- 7. ordering behind an asynchronous process call ----------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_ordered_behind_asynchronous_process_calls(kind):
    N, fs = 64, 96000.0
    cadence = [96, 96]
    F = sum(cadence)
    pairs = 2 if is_q(kind) else 4
    packets = packets_for(kind, N, 7000)
    edits = random_edits(np.random.default_rng(71), kind, np.arange(N), 400)
    a, t = pair(kind, N, F)
    try:
        pcm = torch.from_numpy(pcm_bytes(N, F, 24, 72)).cuda()
        outs_ = {e: (torch.zeros((N, pairs, F, 2), dtype=torch.int32, device="cuda"), torch.zeros((N, F, 8), dtype=torch.int32, device="cuda"))
                 for e in (a, t)}
        for e in (a, t):
            assert not e.apply_bulk_device(packets, fs).any()
        torch.cuda.synchronize()
        for e in (a, t):
            e.process_packets_device(pcm.data_ptr(), 24, cadence, outs_[e][0].data_ptr(), outs_[e][1].data_ptr())
        assert (a.edit_bulk_device(edits, fs) == CURRENT).all()                   # right behind the asynchronous call
        t.sync()
        assert (t.edit_bulk_device(edits, fs) == CURRENT).all()
        for e in (a, t):
            e.process_packets_device(pcm.data_ptr(), 24, cadence, outs_[e][0].data_ptr(), outs_[e][1].data_ptr())
        a.sync()
        t.sync()
        assert torch.equal(outs_[a][0], outs_[t][0]) and torch.equal(outs_[a][1], outs_[t][1])
        assert a.state_export().tobytes() == t.state_export().tobytes()
    finally:
        a.close()
        t.close()


# ---- 8. refusals change nothing -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_refusals_change_nothing(kind):
    N, fs = 6, 48000.0
    packets = packets_for(kind, N, 8000)
    eng, twin = pair(kind, N, 64)
    fn = getattr(api.lib(), eng._PRE + "_edit_bulk_device")
    good = L.bulk_edit(1, ("outputs", 0, "gain_db"), np.float32(-3.0))
    res = np.full(2, 77, np.int32)

    def call(e, handle=True, rate=fs):
        edits = np.concatenate([good, e])                                           # the bad edit is the last one: checked before any write
        return fn(eng._h if handle else None, 2, edits.ctypes.data, 0, float(rate), res.ctypes.data)

    def raw(off, n, inst=0, reserved=0):
        e = np.zeros(1, L.BULK_EDIT)
        e["instance"], e["offset"], e["length"], e["reserved"] = inst, off, n, reserved
        return e

    try:
        for e in (eng, twin):
            assert not e.apply_bulk_device(packets, fs).any()
        img, rec = eng.export_instances().tobytes(), [x.tobytes() for x in eng.collect_bulk_device()]
        assert call(good, handle=False) == EINVAL
        assert fn(eng._h, 1, None, 0, fs, res.ctypes.data) == EINVAL
        for rate in (0.0, -48000.0, float("nan"), float("inf")):
            assert call(good, rate=rate) == EINVAL
        xf = L.edit_field(("crossfeed",))[0]
        for bad in (raw(xf, 0), raw(xf, 25), raw(xf, 4, reserved=1), raw(2896, 5), raw(2899, 2), raw(0, 1), raw(15, 2),
                    raw(L.edit_field(("pins",))[0] - 2, 4), raw(L.edit_field(("eq",))[0] - 1, 2), raw(L.edit_field(("channel_names",))[0], 1),
                    raw(L.edit_field(("i2s_config",))[0] + 15, 2), raw(L.edit_field(("eq",))[0] + 2111, 4)):
            assert call(bad) == EINVAL, bad
        assert call(raw(xf, 4, inst=N)) == ERANGE
        assert call(raw(xf, 4, inst=0xFFFFFFFF)) == ERANGE
        assert fn(eng._h, 0, good.ctypes.data, 0, fs, res.ctypes.data) == 0
        assert (res == 77).all()
        assert eng.export_instances().tobytes() == img and [x.tobytes() for x in eng.collect_bulk_device()] == rec
        assert fn(eng._h, 1, good.ctypes.data, 0, fs, None) == 0       # results may be NULL
        assert (twin.edit_bulk_device(good, fs) == CURRENT).all()
        assert eng.export_instances().tobytes() == twin.export_instances().tobytes()
    finally:
        eng.close()
        twin.close()
