"""Independent float64 model of the engines' frequency response (``dspi_*_response_*``), built from host-side records only:
biquad arrays (``dspi_compute_coefficients_*`` / ``download_biquads``) and CHAIN_PARAMS_F32 / _Q28 records.

Each stage is taken from its recurrence as the oracle states it (oracle/orc_float.inc, oracle/orc_q28.c): a TDF2 band is
(b0 + b1 w + b2 w^2) / (1 + a1 w + a2 w^2), w = z^-1; an SVF band is the transfer function of the 2-state system of
SVF_STEP, computed here as D + w C (I - w A)^-1 B by solving the 2x2 system directly (not through the section
polynomials the GPU uses)."""
import numpy as np

from dspi_b200 import layouts as L

Q28 = 1.0 / (1 << 28)


def _w(freqs, fs):
    return np.exp(-2j * np.pi * (np.asarray(freqs, np.float64) / np.float64(fs)))


def _delay(freqs, fs, d):
    t = np.asarray(freqs, np.float32).astype(np.float64) * float(d) / np.float64(fs)
    t -= np.round(t)
    return np.exp(-2j * np.pi * t)


def _svf(a1, a2, a3, m0, m1, m2, svf_type, general, w):
    """D + w C (I - w A)^-1 B of SVF_STEP (state [ic1, ic2]) with the output mix of svf_type; coefficients may be arrays
    (one per channel, shaped to broadcast against w)."""
    A00, A01, A10, A11 = 2 * a1 - 1, -2 * a2, 2 * a2, 1 - 2 * a3
    B0, B1 = 2 * a2, 2 * a3
    v1c0, v1c1, v1d, v2c0, v2c1, v2d = a1, -a2, a2, a2, 1 - a3, a3
    mixes = {L.LOWPASS: (v2c0, v2c1, v2d),
             L.HIGHPASS: (m1 * v1c0 - v2c0, m1 * v1c1 - v2c1, 1 + m1 * v1d - v2d),
             L.PEAKING: (m1 * v1c0, m1 * v1c1, 1 + m1 * v1d)}
    C0, C1, D = m1 * v1c0 + m2 * v2c0, m1 * v1c1 + m2 * v2c1, m0 + m1 * v1d + m2 * v2d
    if not general:
        for t, (c0, c1, d) in mixes.items():
            sel = np.asarray(svf_type) == t
            C0, C1, D = np.where(sel, c0, C0), np.where(sel, c1, C1), np.where(sel, d, D)
    # (I - w A) x = B, solved per frequency by Cramer's rule
    m00, m01, m10, m11 = 1 - w * A00, -w * A01, -w * A10, 1 - w * A11
    det = m00 * m11 - m01 * m10
    x0 = (B0 * m11 - m01 * B1) / det
    x1 = (m00 * B1 - m10 * B0) / det
    return D + w * (C0 * x0 + C1 * x1)


def _tdf2(b0, b1, b2, a1, a2, w):
    return (b0 + b1 * w + b2 * w * w) / (1 + a1 * w + a2 * w * w)


def band_response(q, w):
    """One record of filters[][] (BIQUAD_F32 or BIQUAD_Q28 scalar); None when bypassed."""
    if int(q["bypass"]):
        return None
    if "use_svf" not in q.dtype.names:
        return _tdf2(*(float(q[k]) * Q28 for k in ("b0", "b1", "b2", "a1", "a2")), w)
    if int(q["use_svf"]):
        return _svf(*(float(q[k]) for k in ("sva1", "sva2", "sva3", "svm0", "svm1", "svm2")), int(q["svf_type"]), False, w)
    return _tdf2(*(float(q[k]) for k in ("b0", "b1", "b2", "a1", "a2")), w)


def row_response(row, n_bands, w):
    h = np.ones_like(w)
    for b in range(n_bands):
        hb = band_response(row[b], w)
        if hb is not None:
            h = h * hb
    return h


def eq_response(biquads, n_bands, freqs, fs):
    """complex128 [C, n_freqs] for biquads [C, 12] (all channels at once)."""
    w = _w(freqs, fs)[None, :]
    h = np.ones((biquads.shape[0], w.size), np.complex128)
    q28 = "use_svf" not in biquads.dtype.names
    with np.errstate(invalid="ignore", divide="ignore"):            # the unselected branch of np.where below
        return _eq_rows(biquads, n_bands, w, h, q28)


def _eq_rows(biquads, n_bands, w, h, q28):
    for b in range(n_bands):
        r = biquads[:, b]
        col = lambda k, s=1.0: r[k].astype(np.float64)[:, None] * s
        if q28:
            hb = _tdf2(*(col(k, Q28) for k in ("b0", "b1", "b2", "a1", "a2")), w)
        else:
            t = _tdf2(*(col(k) for k in ("b0", "b1", "b2", "a1", "a2")), w)
            sv = _svf(*(col(k) for k in ("sva1", "sva2", "sva3", "svm0", "svm1", "svm2")), r["svf_type"][:, None], False, w)
            hb = np.where(r["use_svf"][:, None] != 0, sv, t)
        h = h * np.where(r["bypass"][:, None] != 0, 1.0, hb)
    return h


def _mul_q15(s, g):
    s, g = int(np.int32(s)), int(np.int32(g))
    sh, sl, gh, gl = s >> 16, s & 0xFFFF, g >> 16, g & 0xFFFF
    r = (((sh * gh) & 0xFFFFFFFF) << 17) + (((sh * gl + sl * gh) & 0xFFFFFFFF) << 1) + ((sl * gl) >> 15)
    return int(np.uint32(r & 0xFFFFFFFF).view(np.int32))


def _f2i(x):
    x = float(np.float32(x))
    if x != x:
        return 0
    return int(max(-2147483648, min(2147483647, np.trunc(x))))


def _crossfeed(a0, b1, ap, w):
    lp = a0 / (1 - b1 * w)
    return 1 - lp, (ap + w) / (1 + ap * w) * lp


def chain_response(p, bq, freqs, fs, q28=False, n_bands=L.NUM_BANDS, env_gain=None):
    """complex128 [outputs, 2 inputs, n_freqs] of one instance: CHAIN_PARAMS_F32 / _Q28 record ``p`` and its biquads
    [roles, 12].  ``env_gain``: the envelope's smooth gain when the instance is in envelope mode (else the record's
    constant preset_mute_gain applies)."""
    w = _w(freqs, fs)
    f32 = np.float32
    n_out, max_delay = (L.CHAINQ_OUTPUTS, L.CHAINQ_MAX_DELAY) if q28 else (L.CHAIN_OUTPUTS, L.CHAIN_MAX_DELAY)
    pre = np.ones_like(w)
    if int(p["loudness_enabled"]):
        for j in range(2):
            lc = p["loudness"][j]
            if int(lc["bypass"]):
                continue
            if q28:
                pre = pre * _tdf2(*(float(lc[k]) * Q28 for k in ("b0", "b1", "b2", "a1", "a2")), w)
            else:
                pre = pre * _svf(*(float(lc[k]) for k in ("sva1", "sva2", "sva3", "svm0", "svm1", "svm2")), 0, True, w)
    if int(p["leveller_enabled"]) and int(p["leveller_lookahead"]):
        pre = pre * _delay(freqs, fs, L.LA_SAMPLES)
    master_on = not int(p["bypass_master_eq"])
    P = []
    for s in range(2):
        g = float(p["preamp_q28"][s]) * Q28 if q28 else float(p["preamp_linear"][s])
        h = pre * g
        if master_on:
            h = h * row_response(bq[s], n_bands, w)
        P.append(h)
    direct, cross = np.ones_like(w), np.zeros_like(w)
    if int(p["crossfeed_enabled"]):
        xf = p["crossfeed"]
        k = Q28 if q28 else 1.0
        direct, cross = _crossfeed(float(xf["lp_a0"]) * k, float(xf["lp_b1"]) * k, float(xf["ap_a"]) * k, w)
    # output gain, in the arithmetic of the packet loop (usb_audio.c:569-571 / :975-980)
    gmute = env_gain if env_gain is not None else p["preset_mute_gain"]
    if q28:
        vol = 0 if int(p["host_mute"]) else int(p["host_vol_mul"])
        pmg = int(np.trunc(f32(f32(gmute) * f32(32768.0)) + f32(0.5)))
        pmg = max(0, min(32768, pmg))
        vmm = _mul_q15(_mul_q15(vol, pmg), int(p["master_volume_q15"]))
    else:
        vol = f32(0.0) if int(p["host_mute"]) else f32(int(p["host_vol_mul"])) * f32(1.0 / 32768.0)
        vmm = f32(f32(vol * f32(gmute)) * f32(p["master_volume_linear"]))
    out = np.zeros((n_out, 2, w.size), np.complex128)
    any_delay = any(int(p["matrix"]["outputs"][o]["delay_samples"]) > 0 for o in range(n_out))
    for o in range(n_out):
        oc = p["matrix"]["outputs"][o]
        if not int(oc["enabled"]) or int(oc["mute"]):
            continue
        if q28:
            gain = _f2i(f32(oc["gain_linear"]) * f32(vmm)) / 32768.0
            gx = [(_f2i(f32(-x["gain_linear"] if int(x["phase_invert"]) else x["gain_linear"]) * f32(32768.0)) / 32768.0) if int(x["enabled"]) else 0.0
                  for x in (p["matrix"]["crosspoints"][0, o], p["matrix"]["crosspoints"][1, o])]
        else:
            gain = float(f32(oc["gain_linear"]) * vmm)
            gx = [float(-x["gain_linear"] if int(x["phase_invert"]) else x["gain_linear"]) if int(x["enabled"]) else 0.0
                  for x in (p["matrix"]["crosspoints"][0, o], p["matrix"]["crosspoints"][1, o])]
        if gain == 0.0:
            continue
        g = gain * np.ones_like(w)
        if master_on or not q28:                                    # RP2040: output EQ gated on bypass_master_eq (quirk 3)
            g = g * row_response(bq[2 + o], n_bands, w)
        d = min(max(int(oc["delay_samples"]), 0), max_delay)
        if any_delay and d > 0:
            g = g * _delay(freqs, fs, d & (max_delay - 1))
        out[o, 0] = g * (gx[0] * direct + gx[1] * cross) * P[0]
        out[o, 1] = g * (gx[0] * cross + gx[1] * direct) * P[1]
    return out


def q28_noise_gain(rows, n_bands, T, fs):
    """sum over the active bands of rows (BIQUAD_Q28 [k, 12]) of ||1/A_b||_1 over T samples: every Q28 band truncates its
    products (< 2 LSB each, 5 per sample) and those errors reach the band's output through 1/A(z) - the firmware's
    truncation offsets, which the model does not carry, are bounded by 10 LSB times this gain (times the gain of the
    stages after the band)."""
    w = _w(np.arange(T // 2 + 1) * (fs / T), fs)
    g = 0.0
    for row in rows:
        for b in range(min(n_bands, len(row))):
            r = row[b]
            if int(r["bypass"]):
                continue
            a1, a2 = float(r["a1"]) * Q28, float(r["a2"]) * Q28
            g += np.abs(np.fft.irfft(1.0 / (1 + a1 * w + a2 * w * w), T)).sum()
    return g


def q28_chain_noise_gain(p, bq, T, fs, n_bands=L.NUM_BANDS):
    """q28_noise_gain over every recursive stage of a Q28 chain instance: its EQ rows, the loudness shelves when on and the
    crossfeed low-pass (||1 / (1 - b1 z^-1)||_1 = 1 / (1 - |b1|)) when on."""
    g = q28_noise_gain(bq, n_bands, T, fs)
    if int(p["loudness_enabled"]):
        g += q28_noise_gain([p["loudness"]], 2, T, fs)
    if int(p["crossfeed_enabled"]):
        g += 2.0 / (1.0 - abs(float(p["crossfeed"]["lp_b1"]) * Q28))
    return g
