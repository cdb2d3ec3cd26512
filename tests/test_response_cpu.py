"""The frequency-response model (tests/response_model.py) against the firmware arithmetic, the reference's analytic known
answers on the model, and the argument checks of the six dspi_*_response_* entry points (no GPU needed).

The oracle renders impulse responses long enough to decay.  The model is compared with them in both domains: the rendered
response's DFT against the model on the same T-point grid, and the model's inverse DFT (its impulse response, aliasing
negligible once the response has decayed) against the rendered samples one by one, where the rounding of the path gives a
per-sample bound."""
import ctypes as C

import numpy as np
import pytest

from dspi_b200 import api, layouts as L, workloads as W
from tests import response_model as M
from tests.chain_cases import QUIRK_CASES, chain_params, chain_params_q28, quirk_cases
from tests.orc import make_orc_chain, make_orc_chain_q28, orc_chain_run, orc_chain_run_q28

FS = 48000.0


def _grid(T):
    return np.arange(T // 2 + 1) * (FS / T)


@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
@pytest.mark.parametrize("variant", ["A", "B", "mixed"])
@pytest.mark.parametrize("nb", [1, 2, 7, 10, 11, 12])
def test_eq_model_matches_oracle_impulse_responses(oracle, flavour, variant, nb):
    q = flavour == "q28"
    Cn, T = 6, 1 << 16
    params = W.eq_params(variant, Cn, fs=FS, nbands=L.MAX_BANDS, seed=40 + nb)    # all 12 bands carry a recipe
    bq = api.compute_coefficients(params, q28=q, fs=FS)
    amp = 1 << 27 if q else 1.0                                                     # Q28: half full scale (wraps at 8)
    x = np.zeros((Cn, T), np.int32 if q else np.float32)
    x[:, 0] = amp
    b = bq.copy()
    oracle.eq_many(flavour, b, x, nb, 0)
    h = x.astype(np.float64) / amp
    want = M.eq_response(bq, nb, _grid(T), FS)                                      # bands >= nb excluded
    ir = np.fft.irfft(want, T)
    # per sample: float32 rounding of the cascade, a few 2^-24 of the state magnitudes per band and sample times the
    # sections' noise gain: 1e-4 relative to the peak response.  Q28: every band truncates 5 products per sample (< 2 LSB
    # = 2^-27 each, against an impulse of 2^-1); those errors reach the output through 1/A(z) of their band and the bands
    # after it, so the bound is 10 LSB x sum over bands of ||1/A_b||_1 x prod_(k > b) ||H_k||_1 - for a 31.5 Hz shelf at
    # 48 kHz ||1/A||_1 is about 10^5: the firmware's truncation offset, which the model does not carry.
    tol = 1e-4 * np.maximum(1.0, np.abs(ir).max(axis=1))
    if q:
        grid = _grid(T)
        for c in range(Cn):
            bound, tail = 0.0, 1.0
            for bnd in reversed(range(nb)):
                r = bq[c, bnd]
                if int(r["bypass"]):
                    continue
                a1, a2 = float(r["a1"]) * M.Q28, float(r["a2"]) * M.Q28
                wv = M._w(grid, FS)
                inv_a = np.abs(np.fft.irfft(1.0 / (1 + a1 * wv + a2 * wv * wv), T)).sum()
                bound += 10.0 * 2.0 ** -27 * inv_a * tail
                tail *= np.abs(np.fft.irfft(M.band_response(r, wv), T)).sum()
            tol[c] += bound
    assert np.all(np.abs(h[:, -256:]).max(axis=1) <= (tol if q else 1e-6)), "impulse response has not decayed"
    err = np.abs(h - ir).max(axis=1)
    err_f = np.abs(np.fft.rfft(h, axis=1) - want).max(axis=1)
    print(f"{flavour} {variant} nb={nb}: max |h - ir| / bound {np.max(err / tol):.3g}, max |DFT - H| {err_f.max():.3g}")
    assert np.all(err <= tol)
    # in the DFT: a sum of T per-sample errors
    assert np.all(err_f <= tol * T)


def _impulse_pcm(T, side, amp):
    s = np.zeros((T, 2), np.int32)
    s[0, side] = amp
    b = np.zeros((T, 2, 3), np.uint8)
    b[..., 0] = s & 0xFF
    b[..., 1] = (s >> 8) & 0xFF
    b[..., 2] = (s >> 16) & 0xFF
    return b.reshape(T * 6)


def _render_chain(oracle, flavour, p, bq, T, side, amp):
    """S/PDIF outputs of one instance for an impulse on input `side`, as fractions of the input sample: [outputs - 1, T]."""
    q = flavour == "q28"
    fpp = 128
    pcm = _impulse_pcm(T, side, amp)
    if q:
        words, _ = orc_chain_run_q28(oracle, make_orc_chain_q28(oracle, p, bq), pcm, 24, T // fpp, fpp)
        y = words.astype(np.float64) / amp                                          # (y + 32) >> 6 of Q28 = sample << 6
    else:
        words, _ = orc_chain_run(oracle, flavour, make_orc_chain(oracle, p, bq), pcm, 24, T // fpp, fpp)
        y = words.astype(np.float64) / 8388607.0 / (amp / 8388608.0)
    assert np.abs(words).max() < 0x7FFFFF, "clipped: lower the impulse"
    return y.transpose(0, 2, 1).reshape(-1, T), words


def _chain_cases(oracle, flavour):
    q = flavour == "q28"
    cases = []
    if q:
        P, bq = chain_params_q28(oracle, 6, FS, 71, leveller=False)
    else:
        P, bq = chain_params(oracle, 6, FS, 72, leveller=False)
    cases += [(P[i], bq[i]) for i in range(len(P))]
    for case in QUIRK_CASES:
        if case in ("clipping_hot_input", "pdm_saturation"):
            continue
        p, b, _, _ = quirk_cases(oracle, flavour, case, FS, 192)
        p["leveller_enabled"] = 0
        cases.append((p, b))
    # phase inversions on both inputs, a muted and a disabled output
    p, b = cases[0][0].copy(), cases[0][1].copy()
    m = p["matrix"]
    m["crosspoints"][0, 0]["enabled"], m["crosspoints"][0, 0]["phase_invert"] = 1, 1
    m["crosspoints"][1, 1]["enabled"], m["crosspoints"][1, 1]["phase_invert"] = 1, 1
    m["outputs"][2]["enabled"], m["outputs"][2]["mute"] = 1, 1
    m["outputs"][3]["enabled"] = 0
    cases.append((p, b))
    return cases


@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_chain_model_matches_oracle_impulse_responses(oracle, flavour):
    """Seeded instances (leveller off), the quirk cases (0 dB host-volume polarity flip, dly == MAX and MAX - 1, host mute,
    everything off, sub only), phase inversions, muted and disabled outputs; the RP2040 gate of the output EQs on
    bypass_master_eq comes with the seeded Q28 instances that bypass the master EQ."""
    q = flavour == "q28"
    T = 1 << 15                     # 256 packets of 128 frames; the DFT grid k * 48000 / T is exact in float32, as the GPU takes it
    amp = 1 << 20
    freqs = _grid(T)
    worst = 0.0
    saw = set()
    for p, bq in _chain_cases(oracle, flavour):
        want = M.chain_response(p, bq, freqs, FS, q28=q)
        n_spdif = want.shape[0] - 1
        if int(p["bypass_master_eq"]):
            saw.add("bypass")
        for side in range(2):
            y, _ = _render_chain(oracle, flavour, p, bq, T, side, amp)
            ir = np.fft.irfft(want[:n_spdif, side], T)
            # per sample: the 24-bit word's truncation (float: < 1 LSB) or rounding (Q28: 1/2 LSB plus the Q28 truncation
            # of ~30 products), i.e. about 1.5 LSB of the word relative to the impulse, plus 1e-5 of the peak for the
            # arithmetic's own rounding
            lsb = (1.0 / 8388607.0) / (amp / 8388608.0) if not q else 1.0 / amp
            tol = 1.5 * lsb + 1e-5 * max(1.0, np.abs(ir).max())
            if q:                                                   # 10 LSB of Q28 (impulse = amp << 6) x noise gain x path gain
                tol = tol + 10 * 2.0 ** -28 / (amp * 64 * 2.0 ** -28) * M.q28_chain_noise_gain(p, bq, T, FS) * max(1.0, np.abs(ir).sum(axis=1).max())
            err = np.abs(y - ir).max()
            worst = max(worst, err / tol)
            assert err <= tol, (side, err, tol)
            ok = np.abs(want[:n_spdif, side]).max(axis=1) == 0
            assert np.all(y[ok] == 0), "an output the model calls silent is not"
    print(f"{flavour}: worst per-sample error / bound = {worst:.3f}")
    if q:
        assert "bypass" in saw


def test_known_answers_on_the_model():
    fs = 48000.0
    w1 = np.array([0.0, 100.0, 1000.0, 10000.0, 23999.0])
    # a flat band is the identity (its record is bypassed; a b0 = 1 TDF2 record gives 1 as well)
    flat = np.zeros(1, L.EQ_PARAM)
    flat[0] = (0, 0, L.FLAT, 0, 1000.0, 0.707, 0.0)
    bq = api.compute_coefficients(flat.copy(), fs=fs)
    assert np.array_equal(M.eq_response(np.tile(bq, (1, 12)).reshape(1, 12), 10, w1, fs), np.ones((1, w1.size)))
    rec = bq.copy()
    rec["bypass"] = 0
    assert np.allclose(M.eq_response(np.tile(rec, (1, 12)).reshape(1, 12), 10, w1, fs), 1.0, atol=0, rtol=1e-15)
    # an RBJ peaking band has its set gain at its centre frequency (both topologies, float and Q28)
    for f0 in (1000.0, 12000.0):
        for q28 in (False, True):
            pk = np.zeros((1, 12), L.EQ_PARAM)
            pk["type"] = L.FLAT
            pk[0, 0] = (0, 0, L.PEAKING, 0, f0, 2.0, 4.5)
            b = api.compute_coefficients(pk.copy(), q28=q28, fs=fs)
            g = np.abs(M.eq_response(b, 10, [f0], fs))[0, 0]
            assert abs(20 * np.log10(g) - 4.5) < (1e-3 if q28 else 1e-4), (f0, q28, g)
    # crossfeed: 4.5 dB feed gives G = a0 / (1 - b1) = 0.373 at DC (crossfeed.c:65); a mono input passes at unity at DC;
    # 700 Hz at 48 kHz gives about 217 us of low-pass group delay
    xf = api.crossfeed_coefficients(fs, True, True, 0, 700.0, 4.5)
    direct, cross = M._crossfeed(float(xf["lp_a0"]), float(xf["lp_b1"]), float(xf["ap_a"]), M._w([0.0, 1.0], fs))
    assert abs(cross[0].real - 0.373) < 1e-3 and abs(cross[0].imag) < 1e-12
    assert abs((direct[0] + cross[0]) - 1.0) < 1e-12
    lp = float(xf["lp_a0"]) / (1 - float(xf["lp_b1"]) * M._w([1.0], fs))
    gd = -np.angle(lp[0]) / (2 * np.pi * 1.0)
    assert abs(gd - 217e-6) < 5e-6, gd


@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_full_volume_is_a_polarity_flip_on_the_model(oracle, flavour):
    """quirk 1: 0 dB host volume gives vol_mul = -32768, i.e. gain -1 on every output"""
    p, bq, _, _ = quirk_cases(oracle, flavour, "full_volume_polarity", FS, 192)
    f = np.array([0.0, 440.0, 5000.0])
    h = M.chain_response(p, bq, f, FS, q28=flavour == "q28")
    p2 = p.copy()
    p2["host_vol_mul"] = 16384                                      # +0.5
    h2 = M.chain_response(p2, bq, f, FS, q28=flavour == "q28")
    live = np.abs(h2) > 1e-6
    assert live.any() and np.allclose(h[live] / h2[live], -2.0, rtol=1e-3)


def test_response_entry_points_reject_bad_arguments():
    """dspi_*_response_* check their arguments before any device work: NULL pointers, no or too many frequencies, a
    frequency that is NaN, negative or above Nyquist, a sample rate that is not positive and finite."""
    if not api.os.path.exists(api.LIB_PATH):
        from dspi_b200.build import build
        build()
    lib = api.lib()
    good = np.array([0.0, 100.0, 24000.0], np.float32)
    out = np.zeros(64, np.float32)
    for pre in ("dspi_eq", "dspi_chain", "dspi_chainq"):
        for form in ("_response_host", "_response_device"):
            fn = getattr(lib, pre + form)

            def call(freqs, n_freqs, fs, o=out):
                return fn(None, 0, 1, freqs.ctypes.data if freqs is not None else None, n_freqs, C.c_float(fs),
                          o.ctypes.data if o is not None else None)

            assert call(good, 3, 48000.0) == -22 and b"null argument" in lib.dspi_last_error()     # no engine
            assert call(None, 3, 48000.0) == -22 and b"null frequency" in lib.dspi_last_error()
            assert call(good, 3, 48000.0, None) == -22 and b"null frequency" in lib.dspi_last_error()
            assert call(good, 0, 48000.0) == -22 and b"n_freqs" in lib.dspi_last_error()
            big = np.zeros(65537, np.float32)
            assert call(big, 65537, 48000.0) == -22 and b"n_freqs" in lib.dspi_last_error()
            for fs in (0.0, -48000.0, float("nan"), float("inf")):
                assert call(good, 3, fs) == -22 and b"sample_rate" in lib.dspi_last_error()
            for bad in (float("nan"), -1.0, 24000.5, float("inf")):
                f = good.copy()
                f[1] = bad
                assert call(f, 3, 48000.0) == -22 and b"frequency" in lib.dspi_last_error()
