"""Binary layouts of the records that cross the C-ABI (``include/dspi_b200.h``).

They are byte-for-byte the reference firmware's records so that host configs
drop in unchanged (reference: ``firmware/DSPi/config.h:383-453``,
``crossfeed.h:26-59``, ``leveller.h:59-136``, ``loudness.h:11-23``).  Sizes are
asserted here, in the C header, and against the compiled reference in
``tests/test_oracle_vs_ref.py``.
"""
import numpy as np

MAX_BANDS = 12          # config.h:329  (storage stride of filters[][])
NUM_BANDS = 10          # dsp_pipeline.c:36-44 channel_band_counts
LA_SAMPLES = 480        # leveller.h:36
LOUD_STEPS = 61         # loudness.h:7

FLAT, PEAKING, LOWSHELF, HIGHSHELF, LOWPASS, HIGHPASS = range(6)   # config.h:440-443

_f = np.float32
_i = np.int32
_u = np.uint32
_b = np.uint8

# config.h:418-431 — RP2350 Biquad (68 bytes)
BIQUAD_F32 = np.dtype({
    "names": ["b0", "b1", "b2", "a1", "a2", "s1", "s2", "sva1", "sva2", "sva3",
              "svm0", "svm1", "svm2", "svic1eq", "svic2eq", "svf_type", "use_svf", "bypass"],
    "formats": [_f] * 15 + [_u, _b, _b],
    "offsets": [0, 4, 8, 12, 16, 20, 24, 28, 32, 36, 40, 44, 48, 52, 56, 60, 64, 65],
    "itemsize": 68})

# config.h:433-437, dsp_process_rp2040.S:6-14 — RP2040 Biquad (32 bytes)
BIQUAD_Q28 = np.dtype({
    "names": ["b0", "b1", "b2", "a1", "a2", "s1", "s2", "bypass"],
    "formats": [_i] * 7 + [_b],
    "offsets": [0, 4, 8, 12, 16, 20, 24, 28],
    "itemsize": 32})

# config.h:445-453 — EqParamPacket (packed, 16 bytes)
EQ_PARAM = np.dtype({
    "names": ["channel", "band", "type", "reserved", "freq", "Q", "gain_db"],
    "formats": [_b, _b, _b, _b, _f, _f, _f],
    "offsets": [0, 1, 2, 3, 4, 8, 12],
    "itemsize": 16})

# config.h:383-389 / 392-400 (packed)
CROSSPOINT = np.dtype({
    "names": ["enabled", "phase_invert", "gain_db", "gain_linear"],
    "formats": [_b, _b, _f, _f], "offsets": [0, 1, 4, 8], "itemsize": 12})
OUTPUT = np.dtype({
    "names": ["enabled", "mute", "gain_db", "gain_linear", "delay_ms", "delay_samples"],
    "formats": [_b, _b, _f, _f, _f, _i], "offsets": [0, 1, 4, 8, 12, 16], "itemsize": 20})

# crossfeed.h:46-59 — CrossfeedState (28 bytes)
XFEED_F32 = np.dtype([(n, _f) for n in
                      ("lp_a0", "lp_b1", "lp_state_L", "lp_state_R", "ap_a", "ap_state_L", "ap_state_R")])
XFEED_Q28 = np.dtype([(n, _i) for n in
                      ("lp_a0", "lp_b1", "lp_state_L", "lp_state_R", "ap_a", "ap_state_L", "ap_state_R")])

# leveller.h:81-99 — LevellerCoeffs (36 bytes)
LEV_COEFFS = np.dtype([(n, _f) for n in
                       ("alpha_rms", "alpha_attack", "alpha_release", "threshold_db", "ratio",
                        "knee_width_db", "makeup_db", "gate_threshold_db", "max_gain_db")])
# leveller.h:107-136 — LevellerState (3864 bytes)
LEV_STATE_F32 = np.dtype([("env_sq_l", _f), ("env_sq_r", _f), ("gain_smooth_db", _f),
                          ("gain_linear", _f), ("gain_prev_linear", _f),
                          ("lookahead_buf", _f, (2, LA_SAMPLES)), ("la_write_idx", _u)])
LEV_STATE_Q28 = np.dtype([("env_sq_l", _i), ("env_sq_r", _i), ("gain_smooth_db", _f),
                          ("gain_q28", _i), ("gain_prev_q28", _i),
                          ("lookahead_buf", _i, (2, LA_SAMPLES)), ("la_write_idx", _u)])

# loudness.h:11-23 — LoudnessCoeffs (28 / 24 bytes)
LOUD_F32 = np.dtype({
    "names": ["sva1", "sva2", "sva3", "svm0", "svm1", "svm2", "bypass"],
    "formats": [_f] * 6 + [_b], "offsets": [0, 4, 8, 12, 16, 20, 24], "itemsize": 28})
LOUD_Q28 = np.dtype({
    "names": ["b0", "b1", "b2", "a1", "a2", "bypass"],
    "formats": [_i] * 5 + [_b], "offsets": [0, 4, 8, 12, 16, 20], "itemsize": 24})

# pdm_generator.c:83-87 + loop locals :205-217 (our own packing, 9 words)
PDM_STATE = np.dtype([("err1", _i), ("err2", _i), ("x1", _i), ("x2", _i), ("y1", _i), ("y2", _i),
                      ("err_acc", _i), ("rng", _u), ("fade_in_pos", _u)])

assert BIQUAD_F32.itemsize == 68 and BIQUAD_Q28.itemsize == 32 and EQ_PARAM.itemsize == 16
assert CROSSPOINT.itemsize == 12 and OUTPUT.itemsize == 20
assert XFEED_F32.itemsize == 28 and LEV_COEFFS.itemsize == 36
assert LEV_STATE_F32.itemsize == 3864 and LEV_STATE_Q28.itemsize == 3864
assert LOUD_F32.itemsize == 28 and LOUD_Q28.itemsize == 24 and PDM_STATE.itemsize == 36

# ---- full-chain records (include/dspi_b200.h) ---------------------------------------------------
CHAIN_OUTPUTS = 9
CHAIN_EQ_CHANNELS = 11
CHAIN_MAX_DELAY = 4096

# config.h:403-406 — MatrixMixer, RP2350 (396 bytes)
MATRIX_MIXER_F32 = np.dtype([("crosspoints", CROSSPOINT, (2, CHAIN_OUTPUTS)), ("outputs", OUTPUT, (CHAIN_OUTPUTS,))])
# config.h:455-460 — SystemStatusPacket, RP2350 (26 bytes)
STATUS = np.dtype([("peaks", np.uint16, (CHAIN_EQ_CHANNELS,)), ("cpu0_load", _b), ("cpu1_load", _b), ("clip_flags", np.uint16)])
# dspi_chain_params_f32 (544 bytes)
CHAIN_PARAMS_F32 = np.dtype({
    "names": ["bypass_master_eq", "loudness_enabled", "crossfeed_enabled", "leveller_enabled", "host_mute", "leveller_lookahead",
              "host_vol_mul", "preset_mute_gain", "master_volume_linear", "preamp_linear", "loudness", "crossfeed", "leveller", "matrix"],
    "formats": [_b, _b, _b, _b, _b, _b, np.int16, _f, _f, (_f, (2,)), (LOUD_F32, (2,)), XFEED_F32, LEV_COEFFS, MATRIX_MIXER_F32],
    "offsets": [0, 1, 2, 3, 4, 5, 8, 12, 16, 20, 28, 84, 112, 148],
    "itemsize": 544})
assert MATRIX_MIXER_F32.itemsize == 396 and STATUS.itemsize == 26 and CHAIN_PARAMS_F32.itemsize == 544

# ---- Q28 chain records (RP2040 shape: 2 in -> 5 out) --------------------------------------------
CHAINQ_OUTPUTS = 5
CHAINQ_EQ_CHANNELS = 7
CHAINQ_MAX_DELAY = 2048
MATRIX_MIXER_Q28 = np.dtype([("crosspoints", CROSSPOINT, (2, CHAINQ_OUTPUTS)), ("outputs", OUTPUT, (CHAINQ_OUTPUTS,))])
STATUS_Q28 = np.dtype([("peaks", np.uint16, (CHAINQ_EQ_CHANNELS,)), ("cpu0_load", _b), ("cpu1_load", _b), ("clip_flags", np.uint16)])
CHAIN_PARAMS_Q28 = np.dtype({
    "names": ["bypass_master_eq", "loudness_enabled", "crossfeed_enabled", "leveller_enabled", "host_mute", "leveller_lookahead",
              "host_vol_mul", "preset_mute_gain", "master_volume_q15", "preamp_q28", "loudness", "crossfeed", "leveller", "matrix"],
    "formats": [_b, _b, _b, _b, _b, _b, np.int16, _f, _i, (_i, (2,)), (LOUD_Q28, (2,)), XFEED_Q28, LEV_COEFFS, MATRIX_MIXER_Q28],
    "offsets": [0, 1, 2, 3, 4, 5, 8, 12, 16, 20, 28, 76, 104, 140],
    "itemsize": 360})
assert MATRIX_MIXER_Q28.itemsize == 220 and STATUS_Q28.itemsize == 18 and CHAIN_PARAMS_Q28.itemsize == 360

# ---- bulk parameter packet (bulk_params.h:40-205) and the device state it edits -----------------
WIRE_MAX_CHANNELS, WIRE_MAX_OUTPUTS = 11, 9
PLATFORM_RP2040, PLATFORM_RP2350 = 0, 1
WIRE_BULK = np.dtype([
    ("header", [("format_version", _b), ("platform_id", _b), ("num_channels", _b), ("num_output_channels", _b), ("num_input_channels", _b),
                ("max_bands", _b), ("payload_length", np.uint16), ("fw_version_major", np.uint16), ("fw_version_minor", np.uint16), ("reserved", _u)]),
    ("global", [("preamp_gain_db", _f), ("bypass", _b), ("loudness_enabled", _b), ("reserved", _b, (2,)), ("loudness_ref_spl", _f),
                ("loudness_intensity_pct", _f)]),
    ("crossfeed", [("enabled", _b), ("preset", _b), ("itd_enabled", _b), ("reserved", _b), ("custom_fc", _f), ("custom_feed_db", _f), ("reserved2", _u)]),
    ("legacy", [("gain_db", _f, (3,)), ("mute", _b, (3,)), ("reserved", _b)]),
    ("delays", [("delay_ms", _f, (WIRE_MAX_CHANNELS,))]),
    ("crosspoints", [("enabled", _b), ("phase_invert", _b), ("reserved", _b, (2,)), ("gain_db", _f)], (2, WIRE_MAX_OUTPUTS)),
    ("outputs", [("enabled", _b), ("mute", _b), ("reserved", _b, (2,)), ("gain_db", _f), ("delay_ms", _f)], (WIRE_MAX_OUTPUTS,)),
    ("pins", [("num_pin_outputs", _b), ("pins", _b, (5,)), ("reserved", _b, (2,))]),
    ("eq", [("type", _b), ("reserved", _b, (3,)), ("freq", _f), ("q", _f), ("gain_db", _f)], (WIRE_MAX_CHANNELS, MAX_BANDS)),
    ("channel_names", "S32", (WIRE_MAX_CHANNELS,)),
    ("i2s_config", [("output_types", _b, (4,)), ("bck_pin", _b), ("mck_pin", _b), ("mck_enabled", _b), ("mck_multiplier", _b), ("reserved", _b, (8,))]),
    ("leveller", [("enabled", _b), ("speed", _b), ("lookahead", _b), ("reserved", _b), ("amount", _f), ("max_gain_db", _f), ("gate_threshold_db", _f)]),
    ("preamp", [("preamp_db", _f, (2,)), ("reserved", _b, (8,))]),
    ("master_volume", [("master_volume_db", _f), ("reserved", _b, (12,))]),
])
assert WIRE_BULK.itemsize == 2896

XFEED_CFG = np.dtype({"names": ["enabled", "itd_enabled", "preset", "custom_fc", "custom_feed_db"], "formats": [_b, _b, _b, _f, _f],
                      "offsets": [0, 1, 2, 4, 8], "itemsize": 12})
LEV_CFG = np.dtype({"names": ["enabled", "amount", "speed", "max_gain_db", "lookahead", "gate_threshold_db"], "formats": [_b, _f, _b, _f, _b, _f],
                    "offsets": [0, 4, 8, 12, 16, 20], "itemsize": 24})
# dspi_bulk_state (include/dspi_b200.h): the globals bulk_params_apply() edits
BULK_STATE = np.dtype({
    "names": ["platform", "preamp_db", "preamp_linear", "preamp_q28", "master_volume_db", "master_volume_linear", "master_volume_q15",
              "bypass_master_eq", "loudness_enabled", "loudness_ref_spl", "loudness_intensity_pct", "crossfeed", "leveller",
              "legacy_gain_db", "legacy_gain_linear", "legacy_gain_mul", "legacy_mute", "channel_delays_ms", "crosspoints", "outputs", "recipes"],
    "formats": [_i, (_f, (2,)), (_f, (2,)), (_i, (2,)), _f, _f, _i, _b, _b, _f, _f, XFEED_CFG, LEV_CFG,
                (_f, (3,)), (_f, (3,)), (_i, (3,)), (_b, (3,)), (_f, (WIRE_MAX_CHANNELS,)), (CROSSPOINT, (2, WIRE_MAX_OUTPUTS)),
                (OUTPUT, (WIRE_MAX_OUTPUTS,)), (EQ_PARAM, (WIRE_MAX_CHANNELS, MAX_BANDS))],
    "offsets": [0, 4, 12, 20, 28, 32, 36, 40, 41, 44, 48, 52, 64, 88, 100, 112, 124, 128, 172, 388, 568],
    "itemsize": 2680})

# dspi_preset_mute (include/dspi_b200.h): state of update_preset_mute_envelope(), usb_audio.c:456-498
PRESET_MUTE = np.dtype([("loading", "u1"), ("reserved", "u1", (3,)), ("counter", "<u4"), ("smooth_gain", "<f4")])
assert PRESET_MUTE.itemsize == 12

# dspi_spdif_tx (include/dspi_b200.h): S/PDIF transmitter state of one chain instance, audio_spdif.c:82-88, :372-388
SPDIF_TX = np.dtype([("channel_status", "u1", (5,)), ("block_pos", "u1"), ("reserved", "u1", (2,))])
assert SPDIF_TX.itemsize == 8

# dspi_dynamics_config (include/dspi_b200.h): crossfeed_config + leveller_config + loudness globals + host volume
DYNAMICS_CONFIG = np.dtype([
    ("xf_enabled", "u1"), ("xf_itd_enabled", "u1"), ("xf_preset", "u1"), ("_p0", "u1"), ("xf_custom_fc", "<f4"), ("xf_custom_feed_db", "<f4"),
    ("lev_enabled", "u1"), ("_p1", "u1", (3,)), ("lev_amount", "<f4"), ("lev_speed", "u1"), ("_p2", "u1", (3,)), ("lev_max_gain_db", "<f4"),
    ("lev_lookahead", "u1"), ("_p3", "u1", (3,)), ("lev_gate_threshold_db", "<f4"),
    ("loudness_ref_spl", "<f4"), ("loudness_intensity_pct", "<f4"), ("loudness_enabled", "u1"), ("host_mute", "u1"), ("volume_8_8", "<i2")])
assert DYNAMICS_CONFIG.itemsize == 48

# dspi_bulk_host (include/dspi_b200.h): audio_state of one device beside its bulk packet (apply_bulk_device)
BULK_HOST = np.dtype([("volume_8_8", "<i2"), ("host_mute", "u1"), ("reserved", "u1")])
assert BULK_HOST.itemsize == 4
# DSPI_BULK_*: what collect_bulk_device says of each instance's packet
BULK_CURRENT, BULK_STALE, BULK_UNSET = 0, 1, 2
# dspi_preset_load: per instance, what preset_load() gets from its caller and the preset directory
PRESET_LOAD = np.dtype([("slot_index", "u1"), ("master_volume_mode", "u1"), ("reserved", "u1", (2,)), ("dir_master_volume_db", "<f4")])
assert PRESET_LOAD.itemsize == 8

# dspi_bulk_edit (include/dspi_b200.h): `length` bytes at `offset` of one instance's configuration, in the address space
# WIRE_BULK [0, 2896) followed by BULK_HOST [2896, 2900) (edit_bulk_device)
BULK_EDIT = np.dtype([("instance", "<u4"), ("offset", "<u2"), ("length", "u1"), ("reserved", "u1"), ("bytes", "u1", (24,))])
assert BULK_EDIT.itemsize == 32
BULK_EDIT_SPACE = WIRE_BULK.itemsize + BULK_HOST.itemsize


def edit_field(path):
    """(offset, dtype) of a field of the edit address space, from its path through WIRE_BULK, or through BULK_HOST after
    "host": ``("outputs", 3, "gain_db")``, ``("eq", ch, b)``, ``("crosspoints", side, o)``, ``("host", "volume_8_8")``.
    Integers index array dimensions in order; the offsets are the dtypes' own."""
    path = tuple(path)
    dt, off = (BULK_HOST, WIRE_BULK.itemsize) if path[:1] == ("host",) else (WIRE_BULK, 0)
    shape = ()
    for p in path[1:] if path[:1] == ("host",) else path:
        if isinstance(p, str):
            if shape:
                raise ValueError(f"{path}: {p!r} needs the array index first")
            sub, o = dt.fields[p][:2]
            off += o
            dt, shape = (sub.base, sub.shape) if sub.subdtype else (sub, ())
        else:
            if not shape or not 0 <= int(p) < shape[0]:
                raise ValueError(f"{path}: index {p} out of range")
            shape = shape[1:]
            off += int(p) * int(np.prod(shape, dtype=np.int64)) * dt.itemsize
    return off, (np.dtype((dt, shape)) if shape else dt)


def bulk_edit(instance, path, value):
    """BULK_EDIT [1]: write ``value`` (in the field's own dtype, or raw bytes) into the field at ``path`` (see
    ``edit_field``) of ``instance``."""
    off, dt = edit_field(path)
    raw = bytes(value) if isinstance(value, (bytes, bytearray)) else np.asarray(value, dt).tobytes()
    if not 1 <= len(raw) <= 24 or (not isinstance(value, (bytes, bytearray)) and len(raw) != dt.itemsize):
        raise ValueError(f"{path}: {len(raw)} bytes; an edit carries 1 .. 24 bytes of one field")
    e = np.zeros(1, BULK_EDIT)
    e["instance"], e["offset"], e["length"] = instance, off, len(raw)
    e["bytes"][0, :len(raw)] = np.frombuffer(raw, np.uint8)
    return e
