"""Edits to part of a running engine, checked against the oracle bit for bit: output words, S/PDIF words, PDM bits,
status and downloaded filter state.

A host that serves many device instances changes one channel's or one instance's settings between calls
(dspi_eq_upload_biquads / _download_biquads / _set_params_device with ch0 != 0, dspi_eq_set_param, and
dspi_chain(q)_set_params / _upload_biquads / _download_biquads / _set_eq_params_device / _set_dynamics_device /
_set_preset_mute over [inst0, inst0 + n)).  Those calls index the packed stores at role * N_pad + inst0 in 32- or
64-row groups, so the ranges here start on, end on and straddle group boundaries.  Every channel or instance outside
an edited range must carry on exactly like the oracle of its unchanged settings.

Fresh engines: every band of every channel starts bypassed, as after the firmware's dsp_init_default_filters(), so a
fresh engine passes audio through and a single dspi_eq_set_param gives a one-band EQ.

dspi_chain(q)_reset_state clears leveller, loudness, delay-line, modulator and meter state and keeps filter,
crossfeed and preset-mute envelope state; invalid ranges are refused without touching the engine."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L, workloads as W                                          # noqa: E402
from tests.chain_cases import chain_params, chain_params_q28, pcm_bytes                           # noqa: E402
from tests.orc import arm_mute_envelope, make_orc_chain, make_orc_chain_q28, orc_chain_run, orc_chain_run_q28   # noqa: E402
from tests.test_dynamics_gpu import FS, apply_to_oracle, random_configs                           # noqa: E402
from tests.util import same_bits                                                                  # noqa: E402

GEOMETRY = {1: "tile 32 rows x 64 samples", 2: "tile 64 rows x 32 samples"}
EQ_CASES = [("f32f", 1), ("f32f", 2), ("f32s", 1), ("q28", 1)]
EQ_IDS = ["f32f-cpl1", "f32f-cpl2", "f32s", "q28"]
DSPI_OK, DSPI_EINVAL, DSPI_ERANGE = 0, -22, -34


@pytest.fixture(autouse=True)
def _plain_paths(monkeypatch):
    monkeypatch.delenv("DSPI_JIT", raising=False)
    monkeypatch.delenv("DSPI_DBG", raising=False)
    monkeypatch.delenv("DSPI_F32_CPL", raising=False)


def _default_bank(oracle, q28, rows):
    """[rows, 12] of the record dsp_compute_coefficients() makes of the flat recipe dsp_init_default_filters() sets"""
    p = np.zeros((rows, L.MAX_BANDS), L.EQ_PARAM)
    p["type"], p["freq"], p["Q"] = L.FLAT, 1000.0, 0.707
    p["band"] = np.arange(L.MAX_BANDS, dtype=np.uint8)[None, :]
    bq = np.zeros((rows, L.MAX_BANDS), L.BIQUAD_Q28 if q28 else L.BIQUAD_F32)
    oracle.eq_coeffs(q28, p, bq, FS)
    return bq


# ---- EQ engines -------------------------------------------------------------------------------------------------------
def _eq_engine(monkeypatch, arith, cpl, Cn):
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    eng = api.EqEngine(arith, Cn, 10)
    if arith != "q28":
        assert GEOMETRY[cpl] in eng.kernel_info()
    return eng


def _eq_inputs(arith, Cn, T, k):
    return W.inputs_q28(Cn, T, ch0=4096 * k) if arith == "q28" else W.inputs_f32(Cn, T, ch0=4096 * k)


def _eq_process(eng, x):
    """one whole-engine dspi_eq_process_device over x [C, T] (rows padded to a multiple of 4 elements); returns y"""
    Cn, T = x.shape
    ld = (T + 3) // 4 * 4
    host = np.zeros((Cn, ld), x.dtype)
    host[:, :T] = x
    buf = torch.from_numpy(host).cuda()
    torch.cuda.synchronize()
    eng.process_device(buf.data_ptr(), T, ld)
    eng.sync()
    return buf.cpu().numpy()[:, :T]


def _eq_step(oracle, eng, arith, bank, x, what):
    """process x on the engine and on the oracle bank (updated in place); every channel, output and state, bit for bit"""
    y = _eq_process(eng, x)
    want = x.copy()
    oracle.eq_many(arith, bank, want, 10, 96)
    bad = np.argwhere(y.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, f"{what}: {len(bad)} samples differ from the oracle, channels {sorted(set(bad[:, 0].tolist()))[:12]}"
    st = eng.download()
    assert same_bits(st, bank), f"{what}: filter state differs in channels {sorted(set(np.argwhere(st != bank)[:, 0].tolist()))[:12]}"
    return y, st


FRESH_C, FRESH_T = 100, 295


@pytest.mark.parametrize("arith,cpl", EQ_CASES, ids=EQ_IDS)
def test_fresh_eq_engine_passes_audio_through(monkeypatch, oracle, arith, cpl):
    """No upload: process is the identity, download reports the default record in every band, and one set_param gives
    channel 7 a one-band EQ while every other channel stays the identity"""
    q28 = arith == "q28"
    eng = _eq_engine(monkeypatch, arith, cpl, FRESH_C)
    try:
        x = _eq_inputs(arith, FRESH_C, FRESH_T, 0)
        y = _eq_process(eng, x)
        assert np.array_equal(y.view(np.uint32), x.view(np.uint32)), "a fresh engine must pass audio through"
        st = eng.download()
        assert st["bypass"].all(), "a fresh engine must report every band bypassed"
        bank = _default_bank(oracle, q28, FRESH_C)
        assert same_bits(st, bank), "a fresh engine must hold the record of a flat recipe in every band"
        p = np.zeros(1, L.EQ_PARAM)
        p[0] = (7, 4, L.PEAKING, 0, 2500.0, 2.0, -5.0)
        eng.set_param(7, p[0], FS)
        row = bank[7:8, 4].copy()
        oracle.eq_coeffs(q28, p.copy(), row, FS)
        bank[7, 4] = row[0]
        assert not bank[7]["bypass"][4] and bank[7]["bypass"][np.arange(12) != 4].all()
        x = _eq_inputs(arith, FRESH_C, FRESH_T, 1)
        y, _ = _eq_step(oracle, eng, arith, bank, x, "set_param on a fresh engine")
        others = np.r_[0:7, 8:FRESH_C]
        assert np.array_equal(y[others].view(np.uint32), x[others].view(np.uint32)), "other channels must stay the identity"
        assert np.any(y[7] != x[7]) and np.any(y[7] != 0), "channel 7 must run its one band"
    finally:
        eng.close()


def test_default_record_matches_the_reference(oracle, refs):
    """the default record is what the reference's own dsp_compute_coefficients() makes of dsp_init_default_filters()'s
    flat recipe (every field, both builds)"""
    for q28, ref in ((False, refs["f32s"]), (True, refs["q28"])):
        p = np.zeros((1, L.MAX_BANDS), L.EQ_PARAM)
        p["type"], p["freq"], p["Q"] = L.FLAT, 1000.0, 0.707
        p["band"] = np.arange(L.MAX_BANDS, dtype=np.uint8)[None, :]
        theirs = np.zeros((1, L.MAX_BANDS), L.BIQUAD_Q28 if q28 else L.BIQUAD_F32)
        ref.eq_coeffs(p, theirs, FS)
        assert same_bits(_default_bank(oracle, q28, 1), theirs)


RANGE_C, RANGE_T = 300, 295
EQ_RANGES = [(0, 1), (31, 2), (63, 2), (200, 37), (299, 1)]


@pytest.mark.parametrize("edit", ["upload", "set_params_device", "set_param"])
@pytest.mark.parametrize("arith,cpl", EQ_CASES, ids=EQ_IDS)
def test_eq_coefficient_ranges(monkeypatch, oracle, arith, cpl, edit):
    """300 channels with live state; each range of EQ_RANGES edited, then one whole-engine call.  Edited channels equal
    the oracle with the new records and the carried state, every other channel the oracle of its unchanged bank;
    download(n, ch0) equals the same slice of a whole download."""
    q28 = arith == "q28"
    bank = api.compute_coefficients(W.eq_params("mixed", RANGE_C, fs=FS, seed=51), q28=q28, fs=FS)
    eng = _eq_engine(monkeypatch, arith, cpl, RANGE_C)
    try:
        eng.upload(bank)
        _eq_step(oracle, eng, arith, bank, _eq_inputs(arith, RANGE_C, RANGE_T, 0), "first call")
        for k, (ch0, n) in enumerate(EQ_RANGES):
            rec = W.eq_params("mixed", n, fs=FS, seed=60 + k, ch0=ch0)
            if edit == "upload":
                new = api.compute_coefficients(rec, q28=q28, fs=FS)
                eng.upload(new, ch0=ch0)
                bank[ch0:ch0 + n] = new
            elif edit == "set_params_device":
                got = eng.set_params_device(rec, FS, ch0=ch0)
                sub, want_rec = bank[ch0:ch0 + n].copy(), rec.copy()
                oracle.set_libm_f64(1)                              # the device's libm policy
                try:
                    oracle.eq_coeffs(q28, want_rec, sub, FS)
                finally:
                    oracle.set_libm_f64(0)
                assert got.tobytes() == want_rec.tobytes(), f"({ch0}, {n}): clamped recipes"
                bank[ch0:ch0 + n] = sub
            else:
                for j in range(n):
                    p = rec[j:j + 1, (ch0 + j) % 10].copy()
                    p["band"] = (ch0 + j) % 10
                    eng.set_param(ch0 + j, p[0], FS)
                    row = bank[ch0 + j:ch0 + j + 1, (ch0 + j) % 10].copy()
                    oracle.eq_coeffs(q28, p, row, FS)
                    bank[ch0 + j, (ch0 + j) % 10] = row[0]
            _, st = _eq_step(oracle, eng, arith, bank, _eq_inputs(arith, RANGE_C, RANGE_T, k + 1), f"{edit} ({ch0}, {n})")
            assert same_bits(eng.download(n, ch0), st[ch0:ch0 + n]), f"download({n}, {ch0}) differs from the whole download"
    finally:
        eng.close()


@pytest.mark.parametrize("cpl", [1, 2])
def test_kernel_choice_follows_range_uploads(monkeypatch, oracle, cpl):
    """DSPI_JIT=force: variant A everywhere, then B over [0, 200) in two range calls - the engine must report B's
    signature (B now dominates) - then A again over the same range; bit-exact throughout"""
    monkeypatch.setenv("DSPI_JIT", "force")
    pa = W.eq_params("B", RANGE_C, fs=FS, seed=71)
    pb = pa.copy()
    pb["type"][:, 0] = L.HIGHPASS                                   # band 0: SVF shelf -> SVF high-pass
    bank_a = api.compute_coefficients(pa, q28=False, fs=FS)
    bank_b = api.compute_coefficients(pb, q28=False, fs=FS)
    eng = _eq_engine(monkeypatch, "f32f", cpl, RANGE_C)

    def sig():
        info = eng.kernel_info()
        assert info.startswith("jit sig=0x") and GEOMETRY[cpl] in info, info
        return int(info.split()[1][len("sig="):], 16)

    try:
        eng.upload(bank_a)
        bank = bank_a.copy()
        sig_a = sig()
        _eq_step(oracle, eng, "f32f", bank, _eq_inputs("f32f", RANGE_C, RANGE_T, 0), "variant A")
        for lo, hi in ((0, 120), (120, 200)):
            eng.upload(bank_b[lo:hi], ch0=lo)
            bank[lo:hi] = bank_b[lo:hi]
        sig_b = sig()
        assert sig_b != sig_a and (sig_a ^ sig_b) >> 4 == 0, f"B's signature differs from A's in band 0 only: {sig_a:#x} {sig_b:#x}"
        _eq_step(oracle, eng, "f32f", bank, _eq_inputs("f32f", RANGE_C, RANGE_T, 1), "variant B over [0, 200)")
        for lo, hi in ((0, 120), (120, 200)):
            eng.upload(bank_a[lo:hi], ch0=lo)
            bank[lo:hi] = bank_a[lo:hi]
        assert sig() == sig_a
        _eq_step(oracle, eng, "f32f", bank, _eq_inputs("f32f", RANGE_C, RANGE_T, 2), "variant A again")
    finally:
        eng.close()


# ---- chain engines ----------------------------------------------------------------------------------------------------
NPK, FPP = 4, 96
F_CALL = NPK * FPP


def _chain_engine(monkeypatch, flavour, cpl, N):
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    return api.ChainEngineQ28(N, max_frames=F_CALL) if flavour == "q28" else api.ChainEngine(flavour, N, max_frames=F_CALL)


def _chain_setup(oracle, flavour, N, seed):
    return chain_params_q28(oracle, N, FS, seed) if flavour == "q28" else chain_params(oracle, N, FS, seed)


def _roles(flavour):
    return L.CHAINQ_EQ_CHANNELS if flavour == "q28" else L.CHAIN_EQ_CHANNELS


def _orc_chain(oracle, flavour, p, bq):
    return make_orc_chain_q28(oracle, p, bq) if flavour == "q28" else make_orc_chain(oracle, p, bq)


def _orc_filters(chain, flavour):
    dt = L.BIQUAD_Q28 if flavour == "q28" else L.BIQUAD_F32
    return np.frombuffer(bytes(chain.filters), dt).reshape(11, L.MAX_BANDS)[:_roles(flavour)].copy()


def _orc_set_filters(chain, bq):
    """filters[][] written between packets (main.c:843-856); channel_bypassed follows (dsp_pipeline.c:188-197)"""
    b = np.ascontiguousarray(bq)
    C.memmove(C.addressof(chain.filters), b.ctypes.data, b.nbytes)
    for r in range(b.shape[0]):
        chain.channel_bypassed[r] = 1 if b[r, :10]["bypass"].all() else 0


STATE_FIELDS = ("filters", "channel_bypassed", "loud_state", "levs", "delay_lines", "delay_widx", "pdm", "peaks", "clip_flags",
                "mute_env_on", "preset_loading", "preset_mute_counter", "preset_mute_smooth_gain", "sample_rate_hz")


def _orc_set_params(oracle, flavour, chain, p):
    """the globals of one instance replaced by record p the way the main loop does it, running state kept; the crossfeed
    state comes from the record only when its coefficients differ from the ones in force (crossfeed.c:35-127)"""
    new = _orc_chain(oracle, flavour, p, _orc_filters(chain, flavour))
    for f in STATE_FIELDS:
        setattr(new, f, getattr(chain, f))
    if all(getattr(new.xfeed, f) == getattr(chain.xfeed, f) for f in ("lp_a0", "lp_b1", "ap_a")):
        for f in ("lp_state_L", "lp_state_R", "ap_state_L", "ap_state_R"):
            setattr(new.xfeed, f, getattr(chain.xfeed, f))
    return new


def _orc_run(oracle, flavour, chain, pcm):
    if flavour == "q28":
        return orc_chain_run_q28(oracle, chain, pcm, 24, NPK, FPP)
    return orc_chain_run(oracle, flavour, chain, pcm, 24, NPK, FPP)


def _check_call(oracle, flavour, chains, pcm, out, what):
    spdif, pdm, status = out
    for i, ch in enumerate(chains):
        ws, wp = _orc_run(oracle, flavour, ch, pcm[i])
        assert np.array_equal(spdif[i], ws), f"{what}: instance {i}: S/PDIF words differ from the oracle"
        if ch.out[ch.n_out - 1].enabled:
            assert np.array_equal(pdm[i], wp), f"{what}: instance {i}: PDM bits differ from the oracle"
        n_roles = len(status[i]["peaks"])
        assert list(status[i]["peaks"]) == list(ch.peaks)[:n_roles], f"{what}: instance {i}: peaks"
        assert int(status[i]["clip_flags"]) == int(ch.clip_flags), f"{what}: instance {i}: clip flags"


def _check_filters(flavour, eng, chains, what):
    got = eng.download_biquads()
    for i, ch in enumerate(chains):
        assert same_bits(got[i], _orc_filters(ch, flavour)), f"{what}: instance {i}: downloaded filters differ from the oracle"
    return got


def _call(eng, pcm, k):
    chunk = np.ascontiguousarray(pcm[:, k * F_CALL * 6:(k + 1) * F_CALL * 6])
    return chunk, eng.process_host(chunk, 24, NPK, FPP)


@pytest.mark.parametrize("flavour,cpl", [("f32f", 1), ("f32f", 2), ("q28", 1)], ids=["f32f-cpl1", "f32f-cpl2", "q28"])
def test_fresh_chain_instances_are_bypassed(monkeypatch, oracle, flavour, cpl):
    """N = 70 with biquads uploaded for [10, 30) only: every other instance runs and reports all filter rows bypassed"""
    N = 70
    P, bq = _chain_setup(oracle, flavour, N, 901)
    default = _default_bank(oracle, flavour == "q28", _roles(flavour))
    pcm = pcm_bytes(N, 2 * F_CALL, 24, 902)
    oracle.set_libm_f64(1)
    eng = _chain_engine(monkeypatch, flavour, cpl, N)
    try:
        eng.set_params(P)
        eng.upload_biquads(bq[10:30], inst0=10)
        outside = [i for i in range(N) if not 10 <= i < 30]
        got = eng.download_biquads()
        assert got[outside]["bypass"].all(), "never-uploaded instances must report every band bypassed"
        chains = [_orc_chain(oracle, flavour, P[i], bq[i] if 10 <= i < 30 else default) for i in range(N)]
        for k in range(2):
            chunk, out = _call(eng, pcm, k)
            _check_call(oracle, flavour, chains, chunk, out, f"call {k}")
        _check_filters(flavour, eng, chains, "after two calls")
    finally:
        eng.close()
        oracle.set_libm_f64(0)


@pytest.mark.parametrize("src,dst", [(1, 2), (2, 1)])
def test_fresh_chain_checkpoint_across_geometries(monkeypatch, oracle, src, dst):
    """the same float chain exported under one K1 geometry and imported under the other: instances whose biquads were
    never uploaded stay bypassed and bit-exact"""
    N = 70
    P, bq = _chain_setup(oracle, "f32f", N, 911)
    default = _default_bank(oracle, False, L.CHAIN_EQ_CHANNELS)
    pcm = pcm_bytes(N, 2 * F_CALL, 24, 912)
    oracle.set_libm_f64(1)
    try:
        chains = [_orc_chain(oracle, "f32f", P[i], bq[i] if 10 <= i < 30 else default) for i in range(N)]
        a = _chain_engine(monkeypatch, "f32f", src, N)
        try:
            a.set_params(P)
            a.upload_biquads(bq[10:30], inst0=10)
            chunk, out = _call(a, pcm, 0)
            _check_call(oracle, "f32f", chains, chunk, out, f"call 0 under geometry {src}")
            blob = a.state_export()
        finally:
            a.close()
        b = _chain_engine(monkeypatch, "f32f", dst, N)
        try:
            b.set_params(P)
            b.state_import(blob)
            chunk, out = _call(b, pcm, 1)
            _check_call(oracle, "f32f", chains, chunk, out, f"call 1 resumed under geometry {dst}")
            _check_filters("f32f", b, chains, "after the import")
        finally:
            b.close()
    finally:
        oracle.set_libm_f64(0)


CHAIN_CASES = [("f32f", 1), ("f32f", 2), ("f32s", 1), ("f32s", 2), ("q28", 1)]
CHAIN_IDS = ["f32f-cpl1", "f32f-cpl2", "f32s-cpl1", "f32s-cpl2", "q28"]


def _arm(n):
    st = np.zeros(n, L.PRESET_MUTE)
    st["smooth_gain"] = 1.0
    for k in range(n):
        api.lib().dspi_preset_mute_arm(st[k:k + 1].ctypes.data_as(C.c_void_p), int(FS))
    return st


@pytest.mark.parametrize("flavour,cpl", CHAIN_CASES, ids=CHAIN_IDS)
def test_chain_instance_range_edits(monkeypatch, oracle, flavour, cpl):
    """N = 70 (N_pad 96), three calls of 4 x 96 frames with range edits between them; after every call every instance
    is bit-exact against an oracle instance edited the way the firmware's main loop edits its globals"""
    q28 = flavour == "q28"
    N = 70
    P, bq = _chain_setup(oracle, flavour, N, 921)
    P2, bq2 = _chain_setup(oracle, flavour, N, 922)
    pcm = pcm_bytes(N, 3 * F_CALL, 24, 923)
    oracle.set_libm_f64(1)
    eng = _chain_engine(monkeypatch, flavour, cpl, N)
    try:
        eng.set_params(P)
        eng.upload_biquads(bq)
        chains = [_orc_chain(oracle, flavour, P[i], bq[i]) for i in range(N)]

        def call(k):
            chunk, out = _call(eng, pcm, k)
            _check_call(oracle, flavour, chains, chunk, out, f"call {k}")
            full = _check_filters(flavour, eng, chains, f"call {k}")
            assert same_bits(eng.download_biquads(n=3, inst0=31), full[31:34]), "download_biquads(3, 31) differs from the slice"

        call(0)
        # set_params: volume, matrix gains, delays, mutes and bypass_master_eq change; instance 31 keeps its crossfeed
        # coefficients (running state kept), 32 and 69 get new ones (the record's state)
        for i0, n in ((31, 2), (69, 1)):
            new = P2[i0:i0 + n].copy()
            new["bypass_master_eq"] = 1 - P["bypass_master_eq"][i0:i0 + n]
            new["matrix"]["outputs"]["mute"][:, 1] = 1 - P["matrix"]["outputs"]["mute"][i0:i0 + n, 1]
            new["matrix"]["outputs"]["enabled"][:, 1] = 1
            new["matrix"]["outputs"]["delay_samples"][:, 0] = (P["matrix"]["outputs"]["delay_samples"][i0:i0 + n, 0] + 37) % 1500
            new["matrix"]["crosspoints"]["gain_linear"] *= np.float32(0.75)
            new["host_vol_mul"] = P["host_vol_mul"][i0:i0 + n] // 2
            if i0 == 31:
                new["crossfeed"][0] = P["crossfeed"][31]
            eng.set_params(new, inst0=i0)
            for j in range(n):
                chains[i0 + j] = _orc_set_params(oracle, flavour, chains[i0 + j], new[j])
        for i0, n in ((0, 1), (40, 30)):
            eng.upload_biquads(bq2[i0:i0 + n], inst0=i0)
            for j in range(n):
                _orc_set_filters(chains[i0 + j], bq2[i0 + j])
        rec = np.stack([W.eq_params("mixed", _roles(flavour), fs=FS, seed=930 + i) for i in (63, 64)])
        got = eng.set_eq_params_device(rec, FS, inst0=63)
        for j in range(2):
            filt, r = _orc_filters(chains[63 + j], flavour), rec[j].copy()
            oracle.eq_coeffs(q28, r, filt, FS)
            assert got[j].tobytes() == r.tobytes(), f"instance {63 + j}: clamped recipes"
            _orc_set_filters(chains[63 + j], filt)
        eng.set_preset_mute(_arm(3), FS, inst0=32)
        for i in range(32, 35):
            arm_mute_envelope(chains[i], FS)
        call(1)
        cfgs = random_configs(60, 931)
        eng.set_dynamics_device(cfgs, FS, inst0=5)
        for j in range(60):
            apply_to_oracle(oracle, chains[5 + j], cfgs[j], q28)
        eng.set_preset_mute(None, FS, inst0=33, n=1)                # the constant preset_mute_gain of the record applies again
        chains[33].mute_env_on = 0
        chains[33].preset_mute_gain = float(P["preset_mute_gain"][33])
        call(2)
        env = eng.get_preset_mute()
        for i in (32, 34):
            assert (int(env[i]["loading"]), int(env[i]["counter"])) == (int(chains[i].preset_loading), int(chains[i].preset_mute_counter))
            assert np.float32(env[i]["smooth_gain"]) == np.float32(chains[i].preset_mute_smooth_gain)
    finally:
        eng.close()
        oracle.set_libm_f64(0)


def _orc_reset(oracle, flavour, chain):
    """leveller_reset_state(), the modulator's restart path, loudness shelf state, delay lines, write index and meters"""
    q28 = flavour == "q28"
    (oracle.lib.orc_lev_reset_q28 if q28 else oracle.lib.orc_lev_reset_f32)(C.c_void_p(C.addressof(chain.levs)))
    oracle.lib.orc_pdm_reset(C.c_void_p(C.addressof(chain.pdm)))
    for f in ("loud_state", "delay_lines", "peaks"):
        C.memset(C.addressof(getattr(chain, f)), 0, C.sizeof(getattr(chain, f)))
    chain.delay_widx = 0
    chain.clip_flags = 0


@pytest.mark.parametrize("asynchronous", [False, True], ids=["synced", "after-async-call"])
@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_reset_state(monkeypatch, oracle, flavour, asynchronous):
    """two calls, reset_state(), a third call: equal to oracle instances whose leveller, modulator, loudness, delay and
    meter state was reset and whose filter, crossfeed and preset-mute envelope state was kept.  `after-async-call`: the
    reset is issued right behind an asynchronous process_device, which must still complete on the old state."""
    q28 = flavour == "q28"
    N = 40
    P, bq = _chain_setup(oracle, flavour, N, 941)
    hot = np.arange(N) % 5 == 0                                    # clipping instances: the clip flags must clear
    if q28:
        P["preamp_q28"][hot] = 1 << 30
    else:
        P["preamp_linear"][hot] = 4.0
    P["leveller_enabled"][np.arange(N) % 3 == 0] = 1
    armed = [i for i in range(N) if i % 4 == 2]
    pcm = pcm_bytes(N, 3 * F_CALL, 24, 942)
    oracle.set_libm_f64(1)
    eng = _chain_engine(monkeypatch, flavour, 1, N)
    try:
        eng.set_params(P)
        eng.upload_biquads(bq)
        chains = [_orc_chain(oracle, flavour, P[i], bq[i]) for i in range(N)]
        for i in armed:
            eng.set_preset_mute(_arm(1), FS, inst0=i)
            arm_mute_envelope(chains[i], FS)
        chunk, out = _call(eng, pcm, 0)
        _check_call(oracle, flavour, chains, chunk, out, "call 0")
        chunk = np.ascontiguousarray(pcm[:, F_CALL * 6:2 * F_CALL * 6])
        if asynchronous:
            pairs = 2 if q28 else 4
            st_dt = L.STATUS_Q28 if q28 else L.STATUS
            d_pcm = torch.from_numpy(chunk).cuda()
            d_sp = torch.zeros((N, pairs, F_CALL, 2), dtype=torch.int32, device="cuda")
            d_pdm = torch.zeros((N, F_CALL, 8), dtype=torch.int32, device="cuda")
            d_st = torch.zeros(N * st_dt.itemsize, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            eng.process_device(d_pcm.data_ptr(), 24, NPK, FPP, d_sp.data_ptr(), d_pdm.data_ptr(), d_st.data_ptr())
            eng.reset_state()                                       # no sync in between
            eng.sync()
            out = (d_sp.cpu().numpy(), d_pdm.cpu().numpy().view(np.uint32), np.frombuffer(d_st.cpu().numpy().tobytes(), st_dt))
        else:
            out = eng.process_host(chunk, 24, NPK, FPP)
            eng.reset_state()
        _check_call(oracle, flavour, chains, chunk, out, "call 1")
        assert any(int(out[2][i]["clip_flags"]) for i in np.flatnonzero(hot)), "the hot instances must clip before the reset"
        for ch in chains:
            _orc_reset(oracle, flavour, ch)
        chunk, out = _call(eng, pcm, 2)
        _check_call(oracle, flavour, chains, chunk, out, "call 2, after reset_state")
        _check_filters(flavour, eng, chains, "after reset_state")
        env = eng.get_preset_mute()
        for i in armed:
            assert (int(env[i]["loading"]), int(env[i]["counter"])) == (int(chains[i].preset_loading), int(chains[i].preset_mute_counter))
            assert np.float32(env[i]["smooth_gain"]) == np.float32(chains[i].preset_mute_smooth_gain)
    finally:
        eng.close()
        oracle.set_libm_f64(0)


# ---- argument validation ----------------------------------------------------------------------------------------------
def _bad_ranges(n_total):
    """(first, count) pairs that end past the engine, including one whose end wraps in 32 bits"""
    return [(n_total - 1, 2), (0, n_total + 1), (n_total, 1), (0xFFFFFFFF, 2)]


def _expect(rc, want, what):
    assert rc == want, f"{what}: returned {rc}, expected {want} ({api.lib().dspi_last_error().decode()})"


@pytest.mark.parametrize("arith", ["f32f", "q28"])
def test_eq_range_arguments(monkeypatch, oracle, arith):
    """every range entry point of the EQ engine: a range past the end is DSPI_ERANGE, n = 0 is a no-op, NULL records
    are DSPI_EINVAL - and the next call is byte-identical to an engine that never saw those calls"""
    q28 = arith == "q28"
    Cn, T = 100, 295
    h = api.lib()
    bank = api.compute_coefficients(W.eq_params("mixed", Cn, fs=FS, seed=81), q28=q28, fs=FS)
    a, b = _eq_engine(monkeypatch, arith, 1, Cn), _eq_engine(monkeypatch, arith, 1, Cn)
    try:
        for e in (a, b):
            e.upload(bank)
            _eq_process(e, _eq_inputs(arith, Cn, T, 0))
        garbage = np.full((Cn + 1) * L.MAX_BANDS * bank.dtype.itemsize, 0x7F, np.uint8)     # never read: every call is refused
        params = np.ascontiguousarray(W.eq_params("B", Cn + 1, fs=FS, seed=82))
        out = np.zeros((Cn + 1, L.MAX_BANDS), bank.dtype)
        calls = {
            "upload_biquads": (h.dspi_eq_upload_biquads, garbage.ctypes.data, ()),
            "download_biquads": (h.dspi_eq_download_biquads, out.ctypes.data, ()),
            "set_params_device": (h.dspi_eq_set_params_device, params.ctypes.data, (C.c_float(FS),)),
        }
        for name, (f, ptr, rest) in calls.items():
            def fn(c0, n, p):
                return f(a._h, C.c_uint32(c0), C.c_uint32(n), None if p is None else C.c_void_p(p), *rest)
            for c0, n in _bad_ranges(Cn):
                _expect(fn(c0, n, ptr), DSPI_ERANGE, f"{name}({c0}, {n})")
            _expect(fn(5, 0, ptr), DSPI_OK, f"{name}(5, 0)")
            _expect(fn(0, 1, None), DSPI_EINVAL, f"{name} with NULL records")
        p = np.zeros(1, L.EQ_PARAM)
        p[0] = (0, 4, L.PEAKING, 0, 2500.0, 2.0, -5.0)
        _expect(h.dspi_eq_set_param(a._h, Cn, p.ctypes.data, C.c_float(FS)), DSPI_ERANGE, "set_param past the last channel")
        p["band"] = L.MAX_BANDS
        _expect(h.dspi_eq_set_param(a._h, 0, p.ctypes.data, C.c_float(FS)), DSPI_ERANGE, "set_param band 12")
        _expect(h.dspi_eq_set_param(a._h, 0, None, C.c_float(FS)), DSPI_EINVAL, "set_param with a NULL recipe")
        x = _eq_inputs(arith, Cn, T, 1)
        ya, yb = _eq_process(a, x), _eq_process(b, x)
        assert ya.tobytes() == yb.tobytes(), "refused calls changed the next call's output"
        assert a.download().tobytes() == b.download().tobytes(), "refused calls changed the filter state"
        assert a.kernel_info() == b.kernel_info()
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_chain_range_arguments(monkeypatch, oracle, flavour):
    """every range entry point of a chain engine, as test_eq_range_arguments"""
    q28 = flavour == "q28"
    N = 40
    h = api.lib()
    pre = "dspi_chainq" if q28 else "dspi_chain"
    P, bq = _chain_setup(oracle, flavour, N, 951)
    pcm = pcm_bytes(N, 2 * F_CALL, 24, 952)
    oracle.set_libm_f64(1)
    a, b = _chain_engine(monkeypatch, flavour, 1, N), _chain_engine(monkeypatch, flavour, 1, N)
    try:
        for e in (a, b):
            e.set_params(P)
            e.upload_biquads(bq)
            e.set_preset_mute(_arm(2), FS, inst0=7)
            _call(e, pcm, 0)
        P2, bq2 = _chain_setup(oracle, flavour, N + 1, 953)
        rec = np.ascontiguousarray(np.stack([W.eq_params("B", _roles(flavour), fs=FS, seed=954 + i) for i in range(N + 1)]))
        cfgs = random_configs(N + 1, 955)
        mute = _arm(N + 1)
        dl = np.zeros((N + 1, _roles(flavour), L.MAX_BANDS), bq.dtype)
        gm = np.zeros(N + 1, L.PRESET_MUTE)

        def fn(name):
            f = getattr(h, f"{pre}_{name}")
            return lambda i0, n, p, *rest: f(a._h, C.c_uint32(i0), C.c_uint32(n), None if p is None else C.c_void_p(p), *rest)

        calls = {
            "set_params": (fn("set_params"), P2.ctypes.data, ()),
            "upload_biquads": (fn("upload_biquads"), bq2.ctypes.data, ()),
            "download_biquads": (fn("download_biquads"), dl.ctypes.data, ()),
            "set_eq_params_device": (fn("set_eq_params_device"), rec.ctypes.data, (C.c_float(FS),)),
            "set_dynamics_device": (fn("set_dynamics_device"), cfgs.ctypes.data, (C.c_float(FS),)),
            "set_preset_mute": (fn("set_preset_mute"), mute.ctypes.data, (int(FS),)),
            "get_preset_mute": (fn("get_preset_mute"), gm.ctypes.data, ()),
        }
        for name, (f, ptr, rest) in calls.items():
            for i0, n in _bad_ranges(N):
                _expect(f(i0, n, ptr, *rest), DSPI_ERANGE, f"{name}({i0}, {n})")
                if name == "set_preset_mute":
                    _expect(f(i0, n, None, *rest), DSPI_ERANGE, f"{name}({i0}, {n}, NULL)")
            _expect(f(5, 0, ptr, *rest), DSPI_OK, f"{name}(5, 0)")
            if name != "set_preset_mute":                           # NULL states leave envelope mode there
                _expect(f(0, 1, None, *rest), DSPI_EINVAL, f"{name} with NULL records")
        chunk = np.ascontiguousarray(pcm[:, F_CALL * 6:])
        oa, ob = a.process_host(chunk, 24, NPK, FPP), b.process_host(chunk, 24, NPK, FPP)
        for what, x, y in zip(("S/PDIF words", "PDM bits", "status"), oa, ob):
            assert x.tobytes() == y.tobytes(), f"refused calls changed the next call's {what}"
        assert a.download_biquads().tobytes() == b.download_biquads().tobytes(), "refused calls changed the filter state"
        assert a.get_preset_mute().tobytes() == b.get_preset_mute().tobytes(), "refused calls changed the envelope state"
    finally:
        a.close()
        b.close()
        oracle.set_libm_f64(0)
