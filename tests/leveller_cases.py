"""Signals at controlled leveller-input levels, leveller configurations across the firmware's ranges, settled starting
states and a census of the leveller's block decisions, for the leveller path tests (test_leveller_paths_cpu.py on the
oracle, test_leveller_paths_gpu.py on the engines).

The leveller (leveller.c:148-262, Q28 :275-389) decides once per block (= USB packet) from its RMS envelope: gate, boost,
knee, compression, max-gain clamp; then, per sample, the peak limiter runs while the gain is above unity.  Its RMS
window is 0.1-0.4 s, longer than any run a test can afford through the oracle, so every instance starts from a settled
state instead: the envelope at the mean square of the signal's steady part, the smoothed gain near where that level
puts it, the 480-slot look-ahead ring filled with the 480 frames that precede the compared part and a write index
inside the ring.  The same state goes into the oracle's record and, through the state blob, into the engine.

"level" set: loudness, crossfeed and the master EQ off, preamp 0 dB, so the leveller sees the PCM exactly (float: the
sample / 2^(bits-1); Q28: the sample << (30 - bits), i.e. +6.02 dB against full scale).  "stages" set: the same signals
with those stages on (per-instance variety of tests/chain_cases.py)."""
import ctypes as C

import numpy as np

from dspi_b200 import api, layouts as L
from tests.chain_cases import chain_params, chain_params_q28
from tests.orc import make_orc_chain, make_orc_chain_q28

LA = L.LA_SAMPLES
CEIL = 0.70795                                        # leveller.h:53
INT32_MAX = 2 ** 31 - 1
SPEEDS, AMOUNTS, MAX_GAINS, GATES = (0, 1, 2, 3), (0.0, 50.0, 100.0), (0.0, 15.0, 18.0, 35.0), (-96.0, -60.0, 0.0)
OUTCOMES = ("gate", "boost", "knee", "compression", "clamp", "limiter")

# hand-placed instances, one or more per outcome: (signal, rms dBFS, speed, amount, max_gain_db, gate_db, look-ahead,
# smoothed-gain offset from the settled value in dB)
ANCHORS = [
    ("sine", -50.0, 2, 100.0, 35.0, -96.0, 1, 6.0),   # deep boost past the 35 dB cap: clamp, Q28 gain saturated
    ("bursts", -50.0, 0, 100.0, 35.0, -60.0, 0, 0.0),  # quiet bed, full-scale bursts: limiter at high gain
    ("bursts", -44.0, 1, 50.0, 18.0, -96.0, 1, 0.0),   # limiter behind the look-ahead, cap at the Q28 edge (7.94x)
    ("noise", -20.0, 3, 100.0, 15.0, -60.0, 1, 0.0),   # inside the knee (speed 3 = medium)
    ("noise", -8.0, 2, 50.0, 15.0, -96.0, 0, 0.0),     # compression
    ("sine", -12.0, 2, 100.0, 15.0, -96.0, 0, 12.0),   # compression with a boosted gain left over: attack + limiter
    ("silence", 0.0, 1, 100.0, 15.0, -96.0, 1, 6.0),   # digital silence: gate, gain released to 0 dB
    ("noise", -70.0, 0, 100.0, 35.0, -60.0, 0, 0.0),   # below a -60 dB gate
    ("noise", -30.0, 1, 100.0, 15.0, 0.0, 1, -3.0),    # everything below a 0 dB gate
    ("sine", -40.0, 2, 50.0, 0.0, -96.0, 0, 0.0),      # cap 0 dB: every boost clamped
    ("steps", -26.0, 2, 100.0, 15.0, -96.0, 1, 0.0),   # level steps across the knee
    ("oneside", -10.0, 1, 100.0, 15.0, -96.0, 0, 0.0),  # one side silent, the other loud: stereo-linked RMS and peak
    ("oneside", -36.0, 2, 100.0, 35.0, -96.0, 1, 0.0),
    ("tiny", -95.0, 2, 100.0, 35.0, -96.0, 0, 0.0),    # below the Q28 envelope's quantisation (|s| < 2^14 in Q28)
    ("bursts", -60.0, 2, 100.0, 35.0, -96.0, 1, -6.0),
    ("steps", -26.0, 0, 50.0, 35.0, -60.0, 0, 6.0),
]
SIGNALS = ("sine", "noise", "bursts", "steps", "silence", "tiny", "oneside")
RANDOM_LEVELS = {"sine": (-60.0, -6.0), "noise": (-75.0, -4.0), "bursts": (-60.0, -36.0), "steps": (-30.0, -20.0),
                 "silence": (0.0, 0.0), "tiny": (-100.0, -90.0), "oneside": (-50.0, -6.0)}


def cases(n, seed):
    """n instance cases: the anchors first, then seeded draws over signals, levels and the configuration grid."""
    rng = np.random.default_rng(seed)
    out = [dict(zip(("signal", "level", "speed", "amount", "max_gain", "gate", "lookahead", "offset"), a)) for a in ANCHORS[:n]]
    while len(out) < n:
        sig = SIGNALS[int(rng.integers(len(SIGNALS)))]
        lo, hi = RANDOM_LEVELS[sig]
        out.append(dict(signal=sig, level=float(lo + (hi - lo) * rng.random()), speed=int(rng.integers(4)),
                        amount=float(rng.choice(AMOUNTS, p=[0.2, 0.3, 0.5])), max_gain=float(rng.choice(MAX_GAINS)),
                        gate=float(rng.choice(GATES, p=[0.45, 0.35, 0.2])), lookahead=int(rng.integers(2)),
                        offset=float(rng.choice([-6.0, 0.0, 6.0]))))
    return out


# ---- signals -------------------------------------------------------------------------------------------------------------
def signal(case, F, fs, seed):
    """float64 [LA + F, 2] in [-1, 1) and the settled mean square [2] of its steady part (what the envelope holds)."""
    rng = np.random.default_rng(seed)
    T = LA + F
    t = np.arange(T) / fs
    kind, a = case["signal"], 10.0 ** (case["level"] / 20.0)
    x = np.zeros((T, 2))
    if kind == "sine":
        f = 40.0 + 4000.0 * rng.random()
        ph = 2 * np.pi * rng.random(2)
        x = np.sqrt(2.0) * a * np.sin(2 * np.pi * f * t[:, None] + ph[None, :])
        ms = np.array([a * a, a * a])
    elif kind == "noise":
        x = a * rng.standard_normal((T, 2))
        ms = np.array([a * a, a * a])
    elif kind == "bursts":
        # a quiet noise bed; every 700-1300 frames a 8-32-frame tone burst at 0.5-1.0 of full scale on one or both sides
        x = a * rng.standard_normal((T, 2))
        ms = np.array([a * a, a * a])
        pos = int(rng.integers(100, 600))
        while pos < T:
            m = int(rng.integers(8, 33))
            side = int(rng.integers(3))
            tone = (0.5 + 0.5 * rng.random()) * np.sin(2 * np.pi * (500.0 + 3000.0 * rng.random()) * np.arange(m) / fs + 0.3)
            for s in (0, 1):
                if side == 2 or side == s:
                    x[pos:pos + m, s] = tone[:T - pos]
            pos += int(rng.integers(700, 1300))
    elif kind == "steps":
        # four levels across the knee (-23 .. -17 dB at the float leveller), a new one every quarter of the run
        lv = case["level"] + np.array([0.0, 6.0, 13.0, 3.0])
        seg = np.minimum(np.arange(T) * 4 // T, 3)
        x = (10.0 ** (lv[seg] / 20.0))[:, None] * rng.standard_normal((T, 2))
        ms = np.full(2, 10.0 ** (lv[0] / 10.0))
    elif kind == "silence":
        ms = np.zeros(2)
    elif kind == "tiny":
        x = a * rng.standard_normal((T, 2))
        ms = np.array([a * a, a * a])
    elif kind == "oneside":
        s = int(rng.integers(2))
        x[:, s] = a * rng.standard_normal(T)
        ms = np.zeros(2)
        ms[s] = a * a
    else:
        raise ValueError(kind)
    return np.clip(x, -1.0, 1.0 - 2.0 ** -23), ms


def quantise(x, bit_depth, tiny=False):
    """float [T, 2] -> int32 PCM codes; `tiny` keeps 24-bit codes under 256 (Q28 value < 2^14: mul_q28(s, s) <= 0)."""
    full = float(1 << (bit_depth - 1))
    s = np.clip(np.round(x * full), -full, full - 1).astype(np.int32)
    if tiny and bit_depth == 24:
        s = np.clip(s, -255, 255)
    return s


def pcm_of(s, bit_depth):
    """int32 codes [..., T, 2] -> little-endian packed bytes [..., T * bytes_per_frame]."""
    if bit_depth == 16:
        return np.ascontiguousarray(s.astype("<i2")).view(np.uint8).reshape(s.shape[:-2] + (-1,))
    b = np.zeros(s.shape + (3,), np.uint8)
    b[..., 0], b[..., 1], b[..., 2] = s & 0xFF, (s >> 8) & 0xFF, (s >> 16) & 0xFF
    return b.reshape(s.shape[:-2] + (-1,))


def leveller_input(s, bit_depth, q28):
    """What the leveller sees in the level set: float32 sample / 2^(bits-1), or the Q28 word sample << (30 - bits)."""
    if q28:
        return (s.astype(np.int64) << (30 - bit_depth)).astype(np.int32)
    return (s.astype(np.float64) / float(1 << (bit_depth - 1))).astype(np.float32)


# ---- configurations and settled states ---------------------------------------------------------------------------------
def gain_computer(x_db, threshold, ratio, knee):
    """leveller.c:124-139 in double (the census's classification, not a bit-exact restatement)."""
    half = knee * 0.5
    if x_db > threshold + half:
        return 0.0
    if x_db >= threshold - half:
        d = threshold + half - x_db
        return (1.0 - 1.0 / ratio) * d * d / (2.0 * knee)
    return (threshold - x_db) * (1.0 - 1.0 / ratio)


def settled_gain_db(lc, rms_sq):
    """gc_db of a block whose envelope sits at rms_sq (leveller.c:177-194)."""
    rms_db = 10.0 * np.log10(rms_sq + 1e-30)
    if rms_db < float(lc["gate_threshold_db"]):
        return 0.0
    g = gain_computer(rms_db, float(lc["threshold_db"]), float(lc["ratio"]), float(lc["knee_width_db"])) + float(lc["makeup_db"])
    return min(g, float(lc["max_gain_db"]))


class Instance:
    """One instance: its case, PCM codes [LA + F, 2], settled state and the leveller coefficients of its configuration."""

    def __init__(self, case, fs, F, bit_depth, seed):
        self.case, self.fs, self.bit_depth = case, fs, bit_depth
        x, self.ms = signal(case, F, fs, seed)
        self.s = quantise(x, bit_depth, tiny=case["signal"] == "tiny")
        self.lc = api.leveller_coefficients(fs, case["amount"], case["speed"], case["max_gain"], case["gate"])
        self.la_idx = int(np.random.default_rng(seed + 7).integers(LA))

    @property
    def pre(self):
        return self.s[:LA]

    @property
    def body(self):
        return self.s[LA:]

    def settled(self, q28):
        """LEV_STATE record [1] (float or Q28) this instance starts from."""
        st = np.zeros(1, L.LEV_STATE_Q28 if q28 else L.LEV_STATE_F32)
        scale = 4.0 if q28 else 1.0                       # the Q28 chain sees twice the float level
        ms = self.ms * scale
        if self.case["signal"] == "tiny":                 # a few LSB: the mean square of the codes themselves
            ms = np.mean(leveller_input(self.s, self.bit_depth, False).astype(np.float64) ** 2, axis=0) * scale
        smooth = np.float32(settled_gain_db(self.lc, float(ms.max())) + self.case["offset"])
        gl = np.float32(10.0 ** (float(smooth) / 20.0))
        st["gain_smooth_db"] = smooth
        if q28:
            env = np.minimum(np.floor(ms * 2.0 ** 28), INT32_MAX).astype(np.int32)
            if self.case["signal"] == "tiny":
                env[:] = 0                                 # mul_q28(s, s) of |s| < 2^14 is 0 (s >= 0) or below 0 (s < 0)
            g = int(min(float(gl) * 2.0 ** 28, INT32_MAX))
            st["env_sq_l"], st["env_sq_r"], st["gain_q28"], st["gain_prev_q28"] = env[0], env[1], g, g
        else:
            st["env_sq_l"], st["env_sq_r"], st["gain_linear"], st["gain_prev_linear"] = np.float32(ms[0]), np.float32(ms[1]), gl, gl
        pre = leveller_input(self.pre, self.bit_depth, q28)
        ring = np.roll(pre, self.la_idx, axis=0)           # ring[(idx + k) % LA] = pre[k]: the oldest frame is read first
        st["lookahead_buf"][0] = ring.T
        st["la_write_idx"] = self.la_idx
        return st


def instances(n, fs, F, bit_depth, seed):
    return [Instance(c, fs, F, bit_depth, seed * 1000 + i) for i, c in enumerate(cases(n, seed))]


def params(oracle, q28, insts, fs, seed, stages):
    """(params [N], biquads [N, roles, 12]) with each instance's leveller configuration; `stages` False: loudness,
    crossfeed, master EQ off, preamp and master volume 0 dB, host volume -1 dB, no host mute (the level set)."""
    N = len(insts)
    P, bq = chain_params_q28(oracle, N, fs, seed) if q28 else chain_params(oracle, N, fs, seed)
    P["host_mute"] = 0
    P["preset_mute_gain"] = 1.0
    if not stages:
        P["bypass_master_eq"], P["loudness_enabled"], P["crossfeed_enabled"] = 1, 0, 0
        P["host_vol_mul"] = api.host_volume(-256)[0]       # -1 dB: the words carry the leveller's output at near unity gain
        if q28:
            P["preamp_q28"] = 1 << 28
            P["master_volume_q15"] = 32767
        else:
            P["preamp_linear"] = 1.0
            P["master_volume_linear"] = 1.0
    for i, it in enumerate(insts):
        P[i]["leveller"] = it.lc
        P[i]["leveller_enabled"] = 1
        P[i]["leveller_lookahead"] = it.case["lookahead"]
    return P, bq


# the two level sets the census counts and the GPU tests run: {name: (instances, fs, bit depth, packet lengths, seed)}
LEVEL_SETS = {"level24": (44, 96000.0, 24, [96] * 40, 5), "level16": (44, 48000.0, 16, [48] * 60, 8)}


def make_set(oracle, flavour, n, fs, bit_depth, F, seed, stages=False):
    """(instances, params, biquads, pcm bytes [n, F * bytes_per_frame]) of one set."""
    insts = instances(n, fs, F, bit_depth, seed)
    P, bq = params(oracle, flavour == "q28", insts, fs, seed + 1, stages)
    pcm = np.ascontiguousarray(np.stack([pcm_of(it.body, bit_depth) for it in insts]))
    return insts, P, bq, pcm


def oracle_chain(oracle, q28, p, bq, inst):
    """The oracle instance of record p with inst's settled leveller state."""
    ch = (make_orc_chain_q28 if q28 else make_orc_chain)(oracle, p, bq)
    st = inst.settled(q28)
    C.memmove(C.addressof(ch.levs), st.ctypes.data, st.dtype.itemsize)
    return ch


def levs_record(chain, q28):
    """The oracle instance's LevellerState as a numpy record [1]."""
    dt = L.LEV_STATE_Q28 if q28 else L.LEV_STATE_F32
    return np.frombuffer(C.string_at(C.addressof(chain.levs), dt.itemsize), dt).copy()


# ---- the engine's state blob: leveller sections ------------------------------------------------------------------------
_STATE_MAGIC = 0x53505344


def blob_leveller(blob, q28, N):
    """Writable views into a state blob (dspi_chain(q)_state_export): {field: array [N, ...]} in LEV_STATE terms.
    Sections follow the header in the order of instance_arrays() (chain_host.cuh): loudness state [8][N_pad], crossfeed
    [7][N_pad], the leveller rows (float [5][N_pad]: env_l env_r smooth_db gain gain_prev; Q28 [4][N_pad] env_l env_r
    gain gain_prev, then [1][N_pad] smooth_db), la_write_idx [N_pad], look-ahead ring [2][480][N_pad]."""
    h = np.frombuffer(blob[:40].tobytes(), np.uint32)
    assert h[0] == _STATE_MAGIC and h[3] == N, "not a state blob of this engine"
    hdr = 32 if h[1] == 1 else 40
    Np = (N + 31) // 32 * 32
    w = blob[hdr:].view(np.uint32)                     # every section before the look-ahead ring has 4-byte elements
    o = 15 * Np
    out = {}
    if q28:
        rows = w[o:o + 4 * Np].view(np.int32).reshape(4, Np)
        out["env_sq_l"], out["env_sq_r"], out["gain_q28"], out["gain_prev_q28"] = (rows[k, :N] for k in range(4))
        out["gain_smooth_db"] = w[o + 4 * Np:o + 5 * Np].view(np.float32)[:N]
        ring_dt = np.int32
    else:
        rows = w[o:o + 5 * Np].view(np.float32).reshape(5, Np)
        out["env_sq_l"], out["env_sq_r"], out["gain_smooth_db"], out["gain_linear"], out["gain_prev_linear"] = (rows[k, :N] for k in range(5))
        ring_dt = np.float32
    o += 5 * Np
    out["la_write_idx"] = w[o:o + Np][:N]
    o += Np
    out["lookahead_buf"] = w[o:o + 2 * LA * Np].view(ring_dt).reshape(2, LA, Np)[:, :, :N].transpose(2, 0, 1)
    return out


def write_settled(eng, q28, insts):
    """Every instance's settled leveller state into the engine (state_export, patch, state_import)."""
    blob = eng.state_export().copy()
    v = blob_leveller(blob, q28, len(insts))
    for i, it in enumerate(insts):
        st = it.settled(q28)
        for f in st.dtype.names:
            v[f][i] = st[f][0]
    eng.state_import(blob)


# ---- census --------------------------------------------------------------------------------------------------------------
def classify(lc, st_after, x_out, q28, count):
    """Outcomes of one block from the record after it (st_after) and the samples its per-sample loop saw (x_out [count, 2]:
    the leveller input, delayed by the look-ahead when it is on).  Returns the set of outcomes (plus "saturated" when the
    Q28 gain cast saturated)."""
    if q28:
        el, er = int(st_after["env_sq_l"][0]) / 2.0 ** 28, int(st_after["env_sq_r"][0]) / 2.0 ** 28
    else:
        el, er = float(st_after["env_sq_l"][0]), float(st_after["env_sq_r"][0])
    thr, half = float(lc["threshold_db"]), 0.5 * float(lc["knee_width_db"])
    out = set()
    if max(el, er) + 1e-30 <= 0.0:
        # mul_q28(s, s) of a small negative s is negative (the dropped low product and the floor of >> 12), so the Q28
        # envelope of quiet signals can go below zero: log10 gives NaN, which no branch catches (gc_db NaN)
        out.add("nan")
    elif 10.0 * np.log10(max(el, er) + 1e-30) < float(lc["gate_threshold_db"]):
        out.add("gate")
    else:
        rms_db = 10.0 * np.log10(max(el, er) + 1e-30)
        out.add("boost" if rms_db < thr - half else ("knee" if rms_db <= thr + half else "compression"))
        gc = gain_computer(rms_db, thr, float(lc["ratio"]), float(lc["knee_width_db"])) + float(lc["makeup_db"])
        if gc > float(lc["max_gain_db"]):
            out.add("clamp")
    if q28:
        g0, g1 = int(st_after["gain_prev_q28"][0]) / 2.0 ** 28, int(st_after["gain_q28"][0]) / 2.0 ** 28
        peak = np.abs(x_out.astype(np.float64)).max(axis=1) / 2.0 ** 28
        if int(st_after["gain_q28"][0]) == INT32_MAX:
            out.add("saturated")
    else:
        g0, g1 = float(st_after["gain_prev_linear"][0]), float(st_after["gain_linear"][0])
        peak = np.abs(x_out.astype(np.float64)).max(axis=1)
    g = np.full(count, g1) if count == 1 else g0 + (g1 - g0) * np.arange(count) / (count - 1)
    if np.any((g > 1.0) & (peak * g > CEIL)):
        out.add("limiter")
    return out


def census(oracle, flavour, insts, P, bq, frames):
    """The oracle (its current libm mode) packet by packet over the level set; counts of blocks per outcome, and the
    per-instance outcome sets."""
    q28 = flavour == "q28"
    fn = getattr(oracle.lib, f"orc_{flavour}_chain_packet")
    bd = insts[0].bit_depth
    bpf = 6 if bd == 24 else 4
    counts = {k: 0 for k in OUTCOMES + ("saturated", "nan", "blocks")}
    F = int(sum(frames))
    spdif = np.zeros((2 if q28 else 4, F, 2), np.int32)
    pdm = np.zeros((F, 8), np.uint32)
    for i, it in enumerate(insts):
        ch = oracle_chain(oracle, q28, P[i], bq[i], it)
        data = pcm_of(it.body, bd)
        xin = leveller_input(it.s, bd, q28)
        delayed = xin if it.case["lookahead"] else xin[LA:]
        f0 = 0
        for n in frames:
            fn(C.addressof(ch), data.ctypes.data + f0 * bpf, int(n) * bpf, bd, spdif.ctypes.data + f0 * 8, F * 2, pdm.ctypes.data + f0 * 32)
            after = levs_record(ch, q28)
            for k in classify(it.lc, after, delayed[f0:f0 + n], q28, int(n)):
                counts[k] += 1
            counts["blocks"] += 1
            f0 += int(n)
    return counts
