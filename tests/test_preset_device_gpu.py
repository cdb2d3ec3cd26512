"""GPU: dspi_chain(q)_apply_preset_device / _collect_preset_device - preset slot images (PresetSlot v12) loaded into and
saved from many chain instances on the device (bulk_ingest.cuh).  The expected results come from pieces pinned to the
reference elsewhere: dspi_preset_slot_apply / _collect on the host (byte-identical to flash_storage.c, test_preset_cpu.py),
the bulk route of apply_bulk_device, the recipe clamps of the oracle's coefficient generator, and the policy conversions of
test_bulk_device_gpu.py."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                          # noqa: E402
from tests.bulk_cases import wire_packet                                          # noqa: E402
from tests.chain_cases import pcm_bytes                                           # noqa: E402
from tests.test_bulk_collect_gpu import Shadow, assert_packets, audible, host_records, running   # noqa: E402
from tests.test_bulk_device_gpu import expected, policy_biquads, run_oracle      # noqa: E402
from tests.orc import make_orc_chain, make_orc_chain_q28                           # noqa: E402
from tests.util import load_golden, same_bits                                     # noqa: E402

KINDS = ["f32f", "f32s", "q28"]
EINVAL, ERANGE = -22, -34
OK, ERR_CRC = 0, 3
CURRENT, STALE, UNSET = L.BULK_CURRENT, L.BULK_STALE, L.BULK_UNSET
CHUNK = 1024                                                                      # bulk::kChunk
VERSION_OFFSET, INDEX_OFFSET, CRC_OFFSET, DATA_OFFSET = 4, 6, 8, 12


def is_q(kind):
    return kind == "q28"


def platform(kind):
    return L.PLATFORM_RP2040 if is_q(kind) else L.PLATFORM_RP2350


def engine(kind, n, frames=64):
    return api.ChainEngineQ28(n, max_frames=frames) if is_q(kind) else api.ChainEngine(kind, n, max_frames=frames)


def slot_size(kind):
    return api.preset_slot_size(platform(kind))


def reseal(img, version=None):
    if version is not None:
        img[VERSION_OFFSET:VERSION_OFFSET + 2] = np.frombuffer(np.uint16(version).tobytes(), np.uint8)
    img[CRC_OFFSET:CRC_OFFSET + 4] = np.frombuffer(np.uint32(api.crc32(img[DATA_OFFSET:].tobytes())).tobytes(), np.uint8)
    return img


def padded(images, stride, fill=0xA5):
    out = np.full((images.shape[0], stride), fill, np.uint8)
    out[:, :images.shape[1]] = images
    return out


def source_state(kind, seed, version=6):
    st = api.bulk_state_defaults(platform(kind))
    assert api.bulk_params_apply(audible(wire_packet(platform(kind), seed, version)), st, True) == 0
    return st


def bulk_route(images, slots, modes, dirs, kind):
    """host preset apply -> host bulk collect: the packets the documented host route feeds apply_bulk_device(exact_db = 1)"""
    out, codes = [], []
    for i in range(images.shape[0]):
        st = api.bulk_state_defaults(platform(kind))
        codes.append(api.preset_slot_apply(images[i], int(slots[i]), st, int(modes[i]), float(dirs[i])))
        out.append(api.bulk_params_collect(st))
    return np.concatenate(out), codes


def fixture(kind):
    g = load_golden("preset.npz")
    key = "rp2040" if is_q(kind) else "rp2350"
    as_states = lambda a: np.frombuffer(np.ascontiguousarray(a).tobytes(), L.BULK_STATE).copy()   # noqa: E731
    return as_states(g[f"{key}_state"]), as_states(g[f"{key}_loaded"]), np.ascontiguousarray(g[f"{key}_image"]), g[f"{key}_slot"].astype(np.uint8)


def everything(eng, pcm, npk, fpp):
    """what one process call and the read-back calls show of an engine"""
    sub, pdm, status = eng.process_subframes_host(pcm, 24, [fpp] * npk)
    return [eng.download_biquads(), eng.state_export(), sub, pdm, status, *eng.collect_bulk_device()]


def assert_same_engines(a, b, what=""):
    """records field by field (the padding of a biquad record is not the engine's), everything else byte for byte"""
    for k, (x, y) in enumerate(zip(a, b)):
        same = same_bits(x, y) if x.dtype.names else np.ascontiguousarray(x).tobytes() == np.ascontiguousarray(y).tobytes()
        assert same, f"{what} item {k}"


# ---- 1. the reference's own images --------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_reference_images(oracle, kind):
    fs = 48000.0
    states, loaded, images, slots = fixture(kind)
    n, size, roles = len(states), slot_size(kind), 7 if is_q(kind) else 11
    eng, twin = engine(kind, n), engine(kind, n)
    sh = Shadow(oracle, kind, n)
    try:
        assert list(eng.apply_preset_device(images, fs, slots=slots, master_volume_mode=1, dir_master_volume_db=0.0)) == [OK] * n
        for i in range(n):
            sh.st[i] = loaded[i:i + 1].copy()
            sh.clamp(i, fs)
        got, ghv, marks = eng.collect_bulk_device()
        assert_packets(got, sh.collect(), "loaded fixture:")
        assert (marks == CURRENT).all() and not ghv.view(np.uint8).any()

        packets = np.concatenate([api.bulk_params_collect(states[i:i + 1]) for i in range(n)])
        assert not twin.apply_bulk_device(packets, fs, exact_db=True).any()
        imgs, marks = twin.collect_preset_device(slots)
        assert imgs.shape == (n, size) and (marks == CURRENT).all()
        rec = slice(DATA_OFFSET, DATA_OFFSET + roles * L.MAX_BANDS * 16)
        for i in range(n):
            st = states[i:i + 1].copy()
            before = np.ascontiguousarray(st[0]["recipes"][:roles]).copy()
            one = Shadow(oracle, kind, 1)
            one.st[0] = st
            one.clamp(0, fs)
            assert np.array_equal(imgs[i], api.preset_slot_collect(st, int(slots[i]))), f"instance {i}"
            unclamped = (np.ascontiguousarray(st[0]["recipes"][:roles]).view(np.uint8).reshape(-1, 16) ==
                         before.view(np.uint8).reshape(-1, 16)).all(axis=1)
            assert np.array_equal(imgs[i][:CRC_OFFSET], images[i][:CRC_OFFSET]) and np.array_equal(imgs[i][rec.stop:], images[i][rec.stop:])
            a, b = imgs[i][rec].reshape(-1, 16), images[i][rec].reshape(-1, 16)
            assert np.array_equal(a[unclamped], b[unclamped]), f"instance {i}: unclamped recipes"
    finally:
        eng.close()
        twin.close()


# ---- 2. the bulk route, for gains inside (-120, 80) dB ------------------------------------------------------------------
@pytest.mark.parametrize("stride", ["slot", 4096])
@pytest.mark.parametrize("kind", KINDS)
def test_same_engine_as_the_bulk_route(kind, stride):
    n, fs, npk, fpp = 30, 96000.0, 2, 96
    F = npk * fpp
    rng = np.random.default_rng(200)
    slots = rng.integers(0, 10, n).astype(np.uint8)
    modes = np.arange(n) % 2
    dirs = rng.uniform(-60, 0, n).astype(np.float32)
    versions = [(9, 11, 12)[i % 3] for i in range(n)]
    imgs = np.stack([reseal(api.preset_slot_collect(source_state(kind, 2000 + i), int(slots[i])), versions[i]) for i in range(n)])
    hv = host_records(n, 201)
    packets, codes = bulk_route(imgs, slots, modes, dirs, kind)
    assert codes == [OK] * n
    a, b = running(kind, n, fs, F, 2100)[0], running(kind, n, fs, F, 2100)[0]
    pcm = pcm_bytes(n, 3 * F, 24, 202)
    chunks = [np.ascontiguousarray(pcm[:, k * F * 6:(k + 1) * F * 6]) for k in range(3)]
    try:
        for e in (a, b):
            e.process_subframes_host(chunks[0], 24, [fpp] * npk)
        res = a.apply_preset_device(padded(imgs, slot_size(kind) if stride == "slot" else stride), fs, slots=slots, master_volume_mode=modes,
                                    dir_master_volume_db=dirs, host=hv)
        assert list(res) == [OK] * n
        assert not b.apply_bulk_device(packets, fs, host=hv, exact_db=True).any()
        for k in (1, 2):
            ea, eb = everything(a, chunks[k], npk, fpp), everything(b, chunks[k], npk, fpp)
            assert ea[2].any()
            assert_same_engines(ea, eb, f"process call {k}:")
        assert np.array_equal(a.collect_preset_device(slots)[0], b.collect_preset_device(slots)[0])
        lv = a.collect_bulk_device()[0]["leveller"]
        v9 = np.array(versions) == 9
        assert (lv["amount"][v9] == 50.0).all() and not lv["enabled"][v9].any(), "leveller defaults below version 10"
    finally:
        a.close()
        b.close()


# ---- 3. flash clamps ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_flash_gain_conversion(oracle, kind):
    q28 = is_q(kind)
    gains = [-130.0, -120.0, -119.9, 79.9, 80.0, 95.0]
    mvs = [np.nan, 5.0, -200.0, -6.0, -128.0, -0.5]
    N, npk, fpp, fs = len(mvs), 2, 64, 48000.0
    F = npk * fpp
    no = 5 if q28 else 9
    imgs, sts = [], []
    for i in range(N):
        st = source_state(kind, 3000 + i)
        s = st[0]
        for k, g in enumerate(np.roll(gains, i)):
            s["crosspoints"][k % 2][k % no]["gain_db"] = g
            s["crosspoints"][k % 2][k % no]["enabled"] = 1
            s["outputs"][k % no]["gain_db"] = g
            s["outputs"][k % no]["mute"] = 0
        s["preamp_db"][:] = [gains[i], gains[-1 - i]]
        s["master_volume_db"] = mvs[i]
        s["loudness_enabled"] = 0
        imgs.append(api.preset_slot_collect(st, i))
        sts.append(st)
    imgs = np.stack(imgs)
    hv = np.zeros(N, L.BULK_HOST)
    pcm = pcm_bytes(N, F, 16, 301)
    freqs = np.geomspace(20.0, 20000.0, 24).astype(np.float32)
    oracle.set_libm_f64(1)
    eng, twin, old = engine(kind, N, F), engine(kind, N, F), engine(kind, N, F)
    try:
        base = eng.download_biquads()
        Ps = np.zeros(N, L.CHAIN_PARAMS_Q28 if q28 else L.CHAIN_PARAMS_F32)
        bqs = base.copy()
        packets, codes = bulk_route(imgs, range(N), [1] * N, [0.0] * N, kind)
        assert codes == [OK] * N
        for i in range(N):
            # flash_storage.c's db_to_linear under the libm policy: <= -120 dB -> 0 (a dB value whose policy value is 0),
            # >= 80 dB -> 80 dB; then the derived records as after an exact apply
            w = packets[i:i + 1].copy()
            for f in (w["crosspoints"]["gain_db"], w["outputs"]["gain_db"], w["preamp"]["preamp_db"]):
                f[f <= -120.0] = -1000.0
                f[f >= 80.0] = 80.0
            st = api.bulk_state_defaults(platform(kind))
            rc, P = expected(oracle, st, w, fs, hv[i], True)
            assert rc == 0
            P["matrix"]["crosspoints"]["gain_db"] = packets[i:i + 1]["crosspoints"]["gain_db"][:, :, :no]
            P["matrix"]["outputs"]["gain_db"] = packets[i:i + 1]["outputs"]["gain_db"][:, :no]
            Ps[i], bqs[i] = P[0], policy_biquads(oracle, q28, st, base[i], fs)
            if not q28:
                lin = P[0]["matrix"]["crosspoints"]["gain_linear"].reshape(-1)
                assert (lin[np.isin(w["crosspoints"]["gain_db"][0, :, :no].reshape(-1), [-1000.0])] == 0.0).all()
        mv = packets["master_volume"]["master_volume_db"]
        assert mv[0] == 0.0 and mv[1] == 0.0 and mv[2] == -128.0, "master volume made finite and clamped"
        twin.set_params(Ps)
        twin.upload_biquads(bqs)
        r0 = running(kind, N, fs, F, 3100)                                         # preset-mute gain 1: not the call's to set
        r0[0].close()
        for e in (eng, old):
            e.set_params(r0[1])
        assert list(eng.apply_preset_device(imgs, fs, slots=np.arange(N), master_volume_mode=1, host=hv)) == [OK] * N
        r = eng.response(freqs, fs).view(np.uint32)
        assert np.array_equal(r, twin.response(freqs, fs).view(np.uint32)), "parameter rows"
        assert not old.apply_bulk_device(packets, fs, host=hv, exact_db=True).any()
        assert not np.array_equal(r, old.response(freqs, fs).view(np.uint32)), "the exact conversion of the bulk route differs at the clamps"
        spdif, _, _ = eng.process_host(pcm, 16, npk, fpp)
        for i in range(N):
            ch = (make_orc_chain_q28 if q28 else make_orc_chain)(oracle, Ps[i], bqs[i])
            ws, _ = run_oracle(oracle, kind, ch, pcm[i], 16, npk, fpp)
            assert np.array_equal(spdif[i], ws), f"instance {i}"
    finally:
        for e in (eng, twin, old):
            e.close()
        oracle.set_libm_f64(0)


# ---- 4. coefficients ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fs", [44100.0, 48000.0, 96000.0])
@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_coefficients_match_the_oracle_policy(oracle, kind, fs):
    n, q28 = 37, is_q(kind)
    imgs = np.stack([reseal(api.preset_slot_collect(source_state(kind, 4000 + i), 7), (10, 12)[i % 2]) for i in range(n)])
    eng = engine(kind, n, 96)
    oracle.set_libm_f64(1)
    try:
        base = eng.download_biquads()
        assert not eng.apply_preset_device(imgs, fs, slots=7).any()
        got = eng.download_biquads()
        for i in range(n):
            st = api.bulk_state_defaults(platform(kind))
            assert api.preset_slot_apply(imgs[i], 7, st) == 0
            assert same_bits(got[i], policy_biquads(oracle, q28, st, base[i], fs)), f"instance {i}"
    finally:
        eng.close()
        oracle.set_libm_f64(0)


# ---- 5. rejection -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_rejected_images_change_nothing(oracle, kind):
    fs, size = 48000.0, slot_size(kind)
    good = api.preset_slot_collect(source_state(kind, 5000), 4)
    bad = [good.copy() for _ in range(DATA_OFFSET, size)]
    for k, img in enumerate(bad):                                                 # one bit at every byte the CRC covers
        img[DATA_OFFSET + k] ^= np.uint8(1 << (k % 8))
    for mut in ("crc", "magic", "index"):
        img = good.copy()
        if mut == "crc":
            img[CRC_OFFSET + 2] ^= 0x10
        elif mut == "magic":
            img[1] ^= 0x01
        else:
            img[INDEX_OFFSET] = 5
        bad.append(img)
    bad = np.stack(bad)
    n = bad.shape[0]
    first = np.stack([reseal(api.preset_slot_collect(source_state(kind, 5100 + i % 16), 4), 12) for i in range(n)])
    pcm = pcm_bytes(n, 64, 24, 501)
    r = running(kind, 1, fs, 64, 5200)
    r[0].close()
    eng, twin = engine(kind, n), engine(kind, n)
    try:
        for e in (eng, twin):
            e.set_params(r[1].repeat(n))
            assert not e.apply_preset_device(first[: n // 2], fs, slots=4).any()   # half current, half unset
        assert (eng.apply_preset_device(bad, fs, slots=4) == ERR_CRC).all()
        a, b = everything(eng, pcm, 1, 64), everything(twin, pcm, 1, 64)
        assert_same_engines(a, b, "rejected images:")
        v9 = reseal(good.copy(), 12)
        v9[VERSION_OFFSET] = 9                                                    # outside the CRC: loads with version 9's gates
        assert list(eng.apply_preset_device(v9[None], fs, slots=4, master_volume_mode=1, dir_master_volume_db=-3.0)) == [OK]
        st = api.bulk_state_defaults(platform(kind))
        assert api.preset_slot_apply(v9, 4, st, 1, -3.0) == 0
        got = eng.collect_bulk_device(0, 1)[0]
        assert got["master_volume"]["master_volume_db"][0] == np.float32(-3.0) and got["leveller"]["amount"][0] == 50.0
        sh = Shadow(oracle, kind, 1)
        sh.st[0] = st
        sh.clamp(0, fs)
        assert_packets(got, sh.collect(), "version 9 image:")
    finally:
        eng.close()
        twin.close()


# ---- 6. collect ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_collect_current_stale_unset_and_round_trip(oracle, kind):
    n, fs, npk, fpp, size = 20, 48000.0, 2, 64, slot_size(kind)
    F = npk * fpp
    eng, Ps, _ = running(kind, n, fs, F, 6000)
    twin = running(kind, n, fs, F, 6000)[0]
    slots = (np.arange(n) % 10).astype(np.uint8)
    fn = getattr(api.lib(), eng._PRE + "_collect_preset_device")
    try:
        imgs = np.stack([api.preset_slot_collect(source_state(kind, 6100 + i), int(slots[i])) for i in range(n)])
        hv = host_records(n, 601)
        assert not eng.apply_preset_device(imgs[4:16], fs, inst0=4, slots=slots[4:16], host=hv[4:16]).any()
        eng.set_params(Ps[10:13], inst0=10)                                        # 10..12 stale
        got, marks = eng.collect_preset_device(slots)
        assert list(marks) == [UNSET] * 4 + [CURRENT] * 6 + [STALE] * 3 + [CURRENT] * 3 + [UNSET] * 4
        packets = eng.collect_bulk_device()[0]
        for i in range(n):
            if marks[i] == UNSET:
                assert not got[i].any()
                assert api.preset_slot_apply(got[i], int(slots[i]), api.bulk_state_defaults(platform(kind))) == ERR_CRC
                continue
            st = api.bulk_state_defaults(platform(kind))
            assert api.bulk_params_apply(packets[i:i + 1], st, True) == 0
            assert np.array_equal(got[i], api.preset_slot_collect(st, int(slots[i]))), f"instance {i}"
            assert api.preset_slot_apply(got[i], int(slots[i]), api.bulk_state_defaults(platform(kind)), 1, 0.0) == OK

        buf = np.full((n, 4096), 0x5A, np.uint8)                                   # stride tails are the caller's
        assert fn(eng._h, 0, n, slots.ctypes.data_as(C.c_void_p), buf.ctypes.data_as(C.c_void_p), C.c_size_t(4096), None) == 0
        assert np.array_equal(buf[:, :size], got) and (buf[:, size:] == 0x5A).all()

        cur = marks != UNSET                                                       # the twin as the engine, then the collected images on top
        assert not twin.apply_preset_device(imgs[4:16], fs, inst0=4, slots=slots[4:16], host=hv[4:16]).any()
        assert not twin.apply_preset_device(got[cur], fs, inst0=4, slots=slots[cur], master_volume_mode=1, host=hv[4:16]).any()
        assert np.array_equal(twin.collect_preset_device(slots)[0][cur], got[cur])
        pcm = pcm_bytes(n, F, 24, 602)
        a, b = everything(eng, pcm, npk, fpp), everything(twin, pcm, npk, fpp)
        cur_only = np.nonzero(marks == CURRENT)[0]                                 # a stale instance runs what set_params gave it
        assert_same_engines([x[cur_only] for x in a[:1] + a[2:]], [x[cur_only] for x in b[:1] + b[2:]], "round trip:")

        # behind an asynchronous process call: the configuration in force
        d_pcm = torch.from_numpy(pcm).cuda()
        o = (torch.zeros((n, eng._PAIRS, F, 2), dtype=torch.int32, device="cuda"), torch.zeros((n, F, 8), dtype=torch.int32, device="cuda"),
             torch.zeros(n * eng._STATUS.itemsize, dtype=torch.uint8, device="cuda"))
        torch.cuda.synchronize()
        assert not eng.apply_preset_device(imgs[:4], fs, slots=slots[:4]).any()
        eng.process_device(d_pcm.data_ptr(), 24, npk, fpp, *(t.data_ptr() for t in o))
        again, marks2 = eng.collect_preset_device(slots)
        assert (marks2[:4] == CURRENT).all() and np.array_equal(again[4:], got[4:])
        for i in range(4):
            st = api.bulk_state_defaults(platform(kind))
            assert api.preset_slot_apply(again[i], int(slots[i]), st, 1, 0.0) == OK
        eng.sync()
    finally:
        eng.close()
        twin.close()


# ---- 7. ranges and arguments --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["f32f", "q28"])
def test_ranges_across_the_staging_chunk_and_refused_calls(kind):
    N, inst0, n, fs, size = 2 * CHUNK + 200, 1000, CHUNK + 77, 48000.0, slot_size(kind)
    base = np.stack([api.preset_slot_collect(source_state(kind, 7000 + i), 3) for i in range(16)])
    pick = np.random.default_rng(701).integers(0, 16, n)
    imgs = np.ascontiguousarray(base[pick])
    edge = np.array([CHUNK - 1, CHUNK])                                           # rejected images on both sides of the chunk edge
    imgs[edge, 200] ^= 1
    want_codes = np.zeros(n, np.int32)
    want_codes[edge] = ERR_CRC
    eng = engine(kind, N)
    app = getattr(api.lib(), eng._PRE + "_apply_preset_device")
    col = getattr(api.lib(), eng._PRE + "_collect_preset_device")
    try:
        assert np.array_equal(eng.apply_preset_device(padded(imgs, 4096), fs, inst0=inst0, slots=3), want_codes)
        got, marks = eng.collect_preset_device(3, inst0=inst0 - 3, n=n + 6)
        assert list(marks[:3]) + list(marks[-3:]) == [UNSET] * 6
        assert np.array_equal(marks[3:-3] == UNSET, want_codes != 0)
        ok = np.nonzero(want_codes == 0)[0]
        for k in ok[:: 97]:
            st = api.bulk_state_defaults(platform(kind))
            assert api.preset_slot_apply(got[3 + k], 3, st, 1, 0.0) == OK

        im = np.full(4 * size, 0x5A, np.uint8)
        ld, hv, res, sl = np.zeros(4, L.PRESET_LOAD), np.zeros(4, L.BULK_HOST), np.full(4, 77, np.int32), np.zeros(4, np.uint8)
        p = lambda a: a.ctypes.data_as(C.c_void_p)                                 # noqa: E731
        S = C.c_size_t
        assert app(None, 0, 4, p(im), S(size), p(ld), p(hv), C.c_float(fs), p(res)) == EINVAL
        for k in range(4):
            args = [p(im), S(size), p(ld), p(hv), C.c_float(fs), p(res)]
            args[[0, 2, 3, 5][k]] = None
            assert app(eng._h, 0, 4, *args) == EINVAL
        assert app(eng._h, 0, 4, p(im), S(size - 1), p(ld), p(hv), C.c_float(fs), p(res)) == EINVAL
        for bad_fs in (0.0, -48000.0, float("nan"), float("inf")):
            assert app(eng._h, 0, 4, p(im), S(size), p(ld), p(hv), C.c_float(bad_fs), p(res)) == EINVAL
        assert app(eng._h, N - 3, 4, p(im), S(size), p(ld), p(hv), C.c_float(fs), p(res)) == ERANGE
        assert app(eng._h, 0xFFFFFFFF, 2, p(im), S(size), p(ld), p(hv), C.c_float(fs), p(res)) == ERANGE
        assert app(eng._h, 5, 0, p(im), S(size), p(ld), p(hv), C.c_float(fs), p(res)) == 0
        assert (res == 77).all()
        assert col(None, 0, 4, p(sl), p(im), S(size), p(res)) == EINVAL
        assert col(eng._h, 0, 4, None, p(im), S(size), p(res)) == EINVAL
        assert col(eng._h, 0, 4, p(sl), None, S(size), p(res)) == EINVAL
        assert col(eng._h, 0, 4, p(sl), p(im), S(size - 16), p(res)) == EINVAL
        assert col(eng._h, N - 3, 4, p(sl), p(im), S(size), p(res)) == ERANGE
        assert col(eng._h, 0xFFFFFFFF, 2, p(sl), p(im), S(size), p(res)) == ERANGE
        assert col(eng._h, 5, 0, p(sl), p(im), S(size), p(res)) == 0
        assert (im == 0x5A).all() and (res == 77).all()
        after = eng.collect_preset_device(3, inst0=inst0 - 3, n=n + 6)
        assert np.array_equal(after[0], got) and np.array_equal(after[1], marks), "refused calls changed nothing"
    finally:
        eng.close()
