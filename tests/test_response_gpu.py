"""dspi_*_response_* on the GPU: against the float64 model (tests/response_model.py) for every channel / instance, against
the engines' own processing, after device-side coefficient generation, read-only, in stream order, over partial ranges and
chunked host staging."""
import ctypes as C

import numpy as np
import pytest

from dspi_b200 import api, layouts as L, workloads as W
from tests import response_model as M
from tests.chain_cases import chain_params, chain_params_q28

pytestmark = pytest.mark.gpu

FS = 48000.0
FREQS = np.concatenate([[0.0, FS / 2], np.geomspace(10.0, 23990.0, 62)]).astype(np.float32)   # 64, DC and Nyquist included


def _close(got, want, label):
    """The GPU rounds each double component once to float (2^-24 relative each); the model's own double rounding near
    high-Q poles is bounded by 1e-9 of max(1, |H|)."""
    err = np.abs(got.astype(np.complex128) - want)
    tol = 2.0 ** -23 * np.abs(want) + 1e-9 * np.maximum(1.0, np.abs(want))
    print(f"{label}: max error / bound {np.max(err / tol):.3g}")
    assert np.all(err <= tol), label


def _eq_recipes(Cn, seed):
    """A and B recipes (vectorised generator) with every band type and some bypassed bands mixed in."""
    p = W.eq_params_fast("A", Cn, fs=FS, seed=seed)
    pb = W.eq_params_fast("B", Cn, fs=FS, seed=seed + 1)
    p[1::2] = pb[1::2]
    rng = np.random.default_rng(seed)
    t = p["type"]
    t[:, 2] = rng.integers(0, 6, Cn)                                 # flat / LP / HP / shelves mixed in
    p["type"] = t
    return p


@pytest.mark.parametrize("arith,Cn", [("f32f", 65536), ("f32s", 4096), ("q28", 32768)])
def test_eq_response_matches_model_every_channel(arith, Cn):
    q = arith == "q28"
    e = api.EqEngine(arith, Cn)
    recipes = e.set_params_device(_eq_recipes(Cn, 5), FS)
    bq = e.download()
    got = e.response(FREQS, FS)
    _close(got, M.eq_response(bq, e.n_bands, FREQS, FS), f"{arith} x {Cn}")
    assert recipes.shape == (Cn, L.MAX_BANDS) and (q or np.any(bq["use_svf"]))
    # partial ranges equal the full query; out-of-range requests return DSPI_ERANGE and write nothing
    for ch0, n in ((0, 1), (37, 100), (Cn - 5, 5)):
        assert np.array_equal(e.response(FREQS, FS, ch0, n), got[ch0:ch0 + n])
    out = np.full((2, FREQS.size), 7 + 7j, np.complex64)
    for ch0, n in ((Cn - 1, 2), (0xFFFFFFFF, 2), (Cn, 1)):
        rc = api.lib().dspi_eq_response_host(e._h, ch0, n, FREQS.ctypes.data, FREQS.size, C.c_float(FS), out.ctypes.data)
        assert rc == -34 and np.all(out == 7 + 7j)
    assert e.response(FREQS, FS, 3, 0).shape == (0, FREQS.size)
    e.close()


def _chain_tiled(q, N, D=97):
    """N instances tiled from D (prime) seeded configurations, so a wrong instance index shows."""
    from tests.orc import Oracle
    P, bq = chain_params_q28(Oracle(), D, FS, 11) if q else chain_params(Oracle(), D, FS, 12)
    P["leveller_enabled"][::3] = 1
    idx = np.arange(N) % D
    return P[idx].copy(), bq[idx].copy(), P, bq, idx


@pytest.mark.parametrize("arith", ["f32f", "q28"])
def test_chain_response_matches_model_every_instance(arith):
    q = arith == "q28"
    N = 8192
    P, bq, Pd, bqd, idx = _chain_tiled(q, N)
    ce = api.ChainEngineQ28(N, 192) if q else api.ChainEngine(arith, N, 192)
    ce.set_params(P)
    ce.upload_biquads(bq)
    got = ce.response(FREQS, FS)
    want = np.stack([M.chain_response(Pd[i], bqd[i], FREQS, FS, q28=q) for i in range(len(Pd))])
    _close(got, want[idx], f"{arith} chain x {N}")
    assert np.all(got[:, :, :][~np.any(want[idx] != 0, axis=-1)] == 0)
    for inst0, n in ((0, 1), (4000, 97), (N - 3, 3)):
        assert np.array_equal(ce.response(FREQS, FS, inst0, n), got[inst0:inst0 + n])
    pre = "dspi_chainq" if q else "dspi_chain"
    shape = (2, L.CHAINQ_OUTPUTS if q else L.CHAIN_OUTPUTS, 2, FREQS.size)
    out = np.full(shape, 7 + 7j, np.complex64)
    for inst0, n in ((N - 1, 2), (0xFFFFFFFF, 2)):
        rc = getattr(api.lib(), pre + "_response_host")(ce._h, inst0, n, FREQS.ctypes.data, FREQS.size, C.c_float(FS), out.ctypes.data)
        assert rc == -34 and np.all(out == 7 + 7j)
    ce.close()


def test_host_chunks_equal_the_device_form(monkeypatch):
    import torch
    monkeypatch.setenv("DSPI_HOST_CHUNK_MB", "1")
    f = np.linspace(0.0, FS / 2, 1000).astype(np.float32)
    e = api.EqEngine("f32f", 3000)
    e.set_params_device(_eq_recipes(3000, 9), FS)
    d = torch.empty((3000, f.size), dtype=torch.complex64, device="cuda")
    e.response(f, FS, out_ptr=d.data_ptr())
    e.sync()
    assert np.array_equal(e.response(f, FS), d.cpu().numpy())        # 8 kB rows, 128 per chunk: 24 chunks
    P, bq, _, _, _ = _chain_tiled(False, 300)
    ce = api.ChainEngine("f32f", 300, 192)
    ce.set_params(P)
    ce.upload_biquads(bq)
    d = torch.empty((300, 9, 2, f.size), dtype=torch.complex64, device="cuda")
    ce.response(f, FS, out_ptr=d.data_ptr())
    ce.sync()
    assert np.array_equal(ce.response(f, FS), d.cpu().numpy())      # 144 kB rows, 7 per chunk
    e.close()
    ce.close()


def _impulse_pcm(N, T, side, amp):
    s = np.zeros((N, T, 2), np.int32)
    s[:, 0, side] = amp
    b = np.zeros((N, T, 2, 3), np.uint8)
    for k in range(3):
        b[..., k] = (s >> (8 * k)) & 0xFF
    return b.reshape(N, T * 6)


@pytest.mark.parametrize("arith", ["f32f", "f32s", "q28"])
def test_eq_response_matches_the_engines_own_impulse_responses(arith):
    import torch
    q = arith == "q28"
    Cn, T = 256, 1 << 16
    e = api.EqEngine(arith, Cn)
    e.upload(api.compute_coefficients(W.eq_params("A" if q else "B", Cn, fs=FS, seed=3), q28=q, fs=FS))
    grid = np.arange(T // 2 + 1) * (FS / T)
    H = e.response(grid.astype(np.float32), FS).astype(np.complex128)
    amp = 1 << 27 if q else 1.0
    x = torch.zeros((Cn, T), dtype=torch.int32 if q else torch.float32, device="cuda")
    x[:, 0] = amp
    torch.cuda.synchronize()
    e.process_device(x.data_ptr(), T)
    e.sync()
    h = x.cpu().numpy().astype(np.float64) / amp
    err = np.abs(h - np.fft.irfft(H, T)).max()
    print(f"{arith}: max |impulse response - irfft(H)| = {err:.3g}")
    assert err < 1e-4 * max(1.0, np.abs(h).max())                  # float rounding / Q28 truncation of variant A
    e.close()


@pytest.mark.parametrize("arith", ["f32f", "q28"])
def test_chain_response_matches_the_engines_own_processing(arith):
    """24-bit impulses through process_packets_device (leveller off): the S/PDIF words against irfft of the response.
    Per sample: < 1 LSB of the word's truncation (float) / 1/2 LSB of its rounding plus the Q28 truncation (RP2040),
    relative to the impulse, plus 1e-5 of the peak for the arithmetic's own rounding."""
    import torch
    q = arith == "q28"
    N, fpp, npk, amp = 16, 128, 256, 1 << 20                        # T = 2^15: the DFT grid is exact in float32
    T = fpp * npk
    P, bq, _, _, _ = _chain_tiled(q, N, D=N)
    P["leveller_enabled"] = 0
    grid = (np.arange(T // 2 + 1) * (FS / T)).astype(np.float32)
    pairs = 2 if q else 4
    for side in range(2):
        ce = api.ChainEngineQ28(N, T) if q else api.ChainEngine(arith, N, T)
        ce.set_params(P)
        ce.upload_biquads(bq)
        H = ce.response(grid, FS).astype(np.complex128)
        pcm = torch.from_numpy(_impulse_pcm(N, T, side, amp)).cuda()
        words = torch.zeros((N, pairs, T, 2), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ce.process_packets_device(pcm.data_ptr(), 24, [fpp] * npk, spdif_ptr=words.data_ptr())
        ce.sync()
        w = words.cpu().numpy()
        assert np.abs(w).max() < 0x7FFFFF
        y = w.transpose(0, 1, 3, 2).reshape(N, 2 * pairs, T).astype(np.float64)
        y = y / amp if q else y / 8388607.0 / (amp / 8388608.0)
        ir = np.fft.irfft(H[:, :2 * pairs, side], T)
        lsb = 1.0 / amp if q else (1.0 / 8388607.0) / (amp / 8388608.0)
        err = np.abs(y - ir).max()
        print(f"{arith} side {side}: max error {err:.3g}, 1.5 LSB = {1.5 * lsb:.3g}")
        tol = 1.5 * lsb + 1e-5 * max(1.0, np.abs(ir).max())
        if q:                                                       # Q28 truncation offsets, as in tests/test_response_cpu.py
            tol += max(10 * 2.0 ** -28 / (amp * 64 * 2.0 ** -28) * M.q28_chain_noise_gain(P[i], bq[i], T, FS) for i in range(N)) * max(1.0, np.abs(ir).sum(axis=-1).max())
        assert err <= tol
        ce.close()


def test_known_answers_on_live_engines():
    # an RBJ peaking band generated on the device has its set gain at its centre frequency
    for arith in ("f32f", "q28"):
        e = api.EqEngine(arith, 64)
        r = np.zeros((64, L.MAX_BANDS), L.EQ_PARAM)
        r["type"], r["freq"], r["Q"] = L.FLAT, 1000.0, 0.707
        f0 = np.geomspace(50.0, 15000.0, 64).astype(np.float32)
        r["type"][:, 3], r["freq"][:, 3], r["Q"][:, 3], r["gain_db"][:, 3] = L.PEAKING, f0, 1.5, 5.0
        e.set_params_device(r, FS)
        g = np.array([abs(e.response([f0[c]], FS, c, 1)[0, 0]) for c in range(64)])
        # float32 / Q28 coefficient rounding moves a 50 Hz band's centre gain by a few 1e-4 dB
        assert np.all(np.abs(20 * np.log10(g) - 5.0) < 2e-3), g
        bq = e.download()
        _close(e.response(FREQS, FS), M.eq_response(bq, 10, FREQS, FS), f"{arith} after set_params_device")
        e.close()
    # crossfeed generated on the device with 4.5 dB feed: G = 0.373 at DC, a mono input passes at unity at DC
    ce = api.ChainEngine("f32f", 4, 192)
    P, bq = _chain_tiled(False, 4, D=4)[:2]
    P["bypass_master_eq"], P["loudness_enabled"], P["leveller_enabled"] = 1, 0, 0
    P["preamp_linear"] = 1.0
    xp = P["matrix"]["crosspoints"]
    xp["enabled"][:, 0, 0], xp["phase_invert"][:, 0, 0], xp["gain_linear"][:, 0, 0] = 1, 0, 1.0     # output 1 = L' only
    xp["enabled"][:, 1, 0] = 0
    P["matrix"]["outputs"]["enabled"][:, 0], P["matrix"]["outputs"]["mute"][:, 0] = 1, 0
    bq[:, 2]["bypass"] = 1                                           # Out1's EQ flat
    ce.set_params(P)
    ce.upload_biquads(bq)
    cfg = np.zeros(4, L.DYNAMICS_CONFIG)
    cfg["xf_enabled"], cfg["xf_itd_enabled"], cfg["xf_preset"] = 1, 1, 0        # preset 0: 700 Hz, 4.5 dB feed
    cfg["volume_8_8"] = -6 * 256
    ce.set_dynamics_device(cfg, FS)
    h = ce.response([0.0], FS)[:, 0, :, 0].astype(np.complex128)     # output 1: L' (x gain), from L and from R
    assert np.allclose(h[:, 1] / (h[:, 0] + h[:, 1]), 0.373, atol=1e-3)
    assert np.all(np.abs(h[:, 0] + h[:, 1]) > 0)
    ce.close()


def _setup_pair(q, N=64):
    P, bq, _, _, _ = _chain_tiled(q, N, D=N)
    engines = []
    for _ in range(2):
        ce = api.ChainEngineQ28(N, 384) if q else api.ChainEngine("f32f", N, 384)
        ce.set_params(P)
        ce.upload_biquads(bq)
        st = np.zeros(N // 2, L.PRESET_MUTE)
        st["loading"], st["counter"], st["smooth_gain"] = 1, 700, 1.0
        ce.set_preset_mute(st, int(FS), inst0=N // 4)
        engines.append(ce)
    return engines


@pytest.mark.parametrize("q", [False, True])
def test_response_is_read_only(q):
    from tests.chain_cases import pcm_bytes
    N = 64
    a, b = _setup_pair(q, N)
    pcm = pcm_bytes(N, 292, 24, 4)
    for ce in (a, b):
        ce.process_packets_host(pcm, 24, [192, 100])
    a.response(FREQS, FS)
    import torch
    d = torch.empty((N, 5 if q else 9, 2, FREQS.size), dtype=torch.complex64, device="cuda")
    a.response(FREQS, FS, out_ptr=d.data_ptr())
    assert np.array_equal(a.state_export(), b.state_export())
    assert np.array_equal(a.get_spdif_tx(), b.get_spdif_tx())
    assert np.array_equal(a.get_preset_mute(), b.get_preset_mute())
    pcm = pcm_bytes(N, 288, 24, 6)
    ra, rb = a.process_packets_host(pcm, 24, [96, 192]), b.process_packets_host(pcm, 24, [96, 192])
    for x, y in zip(ra, rb):
        assert np.array_equal(x, y)
    e1, e2 = api.EqEngine("f32f", 256), api.EqEngine("f32f", 256)
    for e in (e1, e2):
        e.upload(api.compute_coefficients(W.eq_params("mixed", 256, fs=FS, seed=2), fs=FS))
    x1, x2 = W.inputs_f32(256, 300), W.inputs_f32(256, 300)
    e1.response(FREQS, FS)
    e1.process_host(x1)
    e2.process_host(x2)
    assert np.array_equal(x1.view(np.uint32), x2.view(np.uint32)) and np.array_equal(e1.download(), e2.download())


@pytest.mark.parametrize("q", [False, True])
def test_response_follows_the_engine_stream(q):
    """A response issued right behind an asynchronous process call sees the preset-mute gain that call reached."""
    import torch
    from tests.chain_cases import pcm_bytes
    N = 64
    ce, other = _setup_pair(q, N)
    other.close()
    P, bq, _, _, _ = _chain_tiled(q, N, D=N)
    pcm = torch.from_numpy(pcm_bytes(N, 96, 24, 5)).cuda()
    d = torch.empty((N, 5 if q else 9, 2, FREQS.size), dtype=torch.complex64, device="cuda")
    torch.cuda.synchronize()
    ce.process_packets_device(pcm.data_ptr(), 24, [64, 32])           # a fade over 384 frames: 1/4 of it
    ce.response(FREQS, FS, out_ptr=d.data_ptr())                     # no sync in between
    ce.sync()
    got = d.cpu().numpy()
    g = ce.get_preset_mute()["smooth_gain"]
    assert np.any((g > 0) & (g < 1))                                  # fades in progress
    for i in range(N):
        env = float(g[i]) if N // 4 <= i < N // 4 + N // 2 else None
        _close(got[i], M.chain_response(P[i], bq[i], FREQS, FS, q28=q, env_gain=env), f"instance {i}")
    ce.close()
