"""S/PDIF subframes straight from the chain engines' output stage (dspi_chain(q)_process_subframes_*) and the per-instance
transmitter state (dspi_chain(q)_get/set_spdif_tx): bit for bit against the oracle's encoder over the oracle chain's words,
and against the two-pass path (the words form followed by dspi_spdif_encode_*)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L, workloads as W                                  # noqa: E402
from tests.chain_cases import chain_params, chain_params_q28, pcm_bytes                  # noqa: E402
from tests.orc import make_orc_chain, make_orc_chain_q28                                 # noqa: E402
from tests.util import load_golden                                                       # noqa: E402

CADENCE_44K1 = [44] * 9 + [45]
CALLS = [[96, 96, 96], CADENCE_44K1, [48, 47, 49, 48, 48, 49, 47, 48, 49]]   # 288, 441 and 433 frames: positions wrap
DEFAULT_CS = bytes(api.SPDIF_CHANNEL_STATUS)
# (flavour, K1 geometry of the float engines): fused and strict under both DSPI_F32_CPL values, and the Q28 chain
ENGINES = [("f32f", "1"), ("f32f", "2"), ("f32s", "1"), ("f32s", "2"), ("q28", None)]
ENGINE_IDS = ["f32f-cpl1", "f32f-cpl2", "f32s-cpl1", "f32s-cpl2", "q28"]


@pytest.fixture
def make_engine(monkeypatch):
    """make_engine(flavour, N, F, cpl=None): an engine created under DSPI_F32_CPL = cpl (float only); closed after the test."""
    made = []

    def make(flavour, N, F, cpl=None):
        if cpl is None:
            monkeypatch.delenv("DSPI_F32_CPL", raising=False)
        else:
            monkeypatch.setenv("DSPI_F32_CPL", cpl)
        e = api.ChainEngineQ28(N, max_frames=F) if flavour == "q28" else api.ChainEngine(flavour, N, max_frames=F)
        made.append(e)
        return e

    yield make
    for e in made:
        e.close()


@pytest.fixture
def libm_f64(oracle):
    """the leveller's per-block libm in double on the oracle side too, as the engines run it"""
    oracle.set_libm_f64(1)
    yield oracle
    oracle.set_libm_f64(0)


def _pairs(flavour):
    return 2 if flavour == "q28" else 4


def _config(oracle, flavour, N, fs, seed):
    """the seeded chain config, plus: a muted output, a pair with both outputs disabled, hot inputs that clip, and delays"""
    P, bq = chain_params_q28(oracle, N, fs, seed) if flavour == "q28" else chain_params(oracle, N, fs, seed)
    n_out = 5 if flavour == "q28" else 9
    for i in range(N):
        m = P[i]["matrix"]["outputs"]
        if i % 5 == 0:
            m[0]["mute"] = 1
        if i % 5 == 1:
            m[2]["enabled"], m[3]["enabled"] = 0, 0
        if i % 3 == 2:
            for o in range(n_out):
                m[o]["delay_samples"] = [0, 1, 7, 50, 97, 200, 333, 450, 1000][o]
    hot = np.arange(N) % 4 == 3
    if flavour == "q28":
        P["preamp_q28"][hot] = 1 << 30                      # +12 dB
    else:
        P["preamp_linear"][hot] = 4.0
    return P, bq


def _tx(N, seed):
    """per-instance block positions (0, 1 and 191 among them) and channel status (byte 3, the rate code, varies)"""
    rng = np.random.default_rng(seed)
    bp = rng.integers(0, 192, N)
    bp[:3] = [0, 1, 191]
    cs = np.tile(np.frombuffer(DEFAULT_CS, np.uint8), (N, 1))
    cs[:, 3] = np.arange(N) % 16
    cs[::7, 0] = 0x05                                      # a few instances with another byte 0
    return bp, cs


def _orc_words(oracle, flavour, chain, pcm, bit_depth, frames):
    """the oracle chain, one process_audio_packet() per packet; S/PDIF words [pairs, F, 2]"""
    F, bpf = int(sum(frames)), (6 if bit_depth == 24 else 4)
    spdif = np.zeros((_pairs(flavour), F, 2), np.int32)
    pdm = np.zeros((F, 8), np.uint32)
    fn = getattr(oracle.lib, "orc_q28_chain_packet" if flavour == "q28" else f"orc_{flavour}_chain_packet")
    data = np.ascontiguousarray(pcm)
    f0 = 0
    for k in frames:
        fn(C.addressof(chain), data.ctypes.data + f0 * bpf, int(k) * bpf, bit_depth, spdif.ctypes.data + f0 * 8, F * 2, pdm.ctypes.data + f0 * 32)
        f0 += int(k)
    return spdif


def _setup(eng, P, bq):
    eng.set_params(P)
    eng.upload_biquads(bq)


def _chunks(pcm, calls, bpf):
    f0 = 0
    for frames in calls:
        F = int(sum(frames))
        yield frames, np.ascontiguousarray(pcm[:, f0 * bpf:(f0 + F) * bpf])
        f0 += F


def _two_pass(words, bp, cs):
    """dspi_spdif_encode_host over every instance's words at that instance's position and status"""
    return np.stack([api.spdif_encode_host(words[i], int(bp[i]), bytes(cs[i])) for i in range(words.shape[0])])


def _check_tx(eng, bp, cs):
    got = eng.get_spdif_tx()
    assert np.array_equal(got["block_pos"], np.asarray(bp) % 192)
    assert np.array_equal(got["channel_status"], cs)


# ---- 1. fused output == oracle encoder over the oracle's words == two-pass path ----------------------------------------------
@pytest.mark.parametrize("flavour,cpl", ENGINES, ids=ENGINE_IDS)
def test_fused_equals_oracle_and_two_pass(libm_f64, make_engine, flavour, cpl):
    oracle = libm_f64
    N, fs, bd = 70, 48000.0, 24
    P, bq = _config(oracle, flavour, N, fs, 810)
    bp, cs = _tx(N, 811)
    F_max = max(sum(c) for c in CALLS)
    pcm = pcm_bytes(N, sum(sum(c) for c in CALLS), bd, 812)
    eng, twin = make_engine(flavour, N, F_max, cpl), make_engine(flavour, N, F_max, cpl)
    for e in (eng, twin):
        _setup(e, P, bq)
    eng.set_spdif_tx(bp, cs)
    chains = [(make_orc_chain_q28 if flavour == "q28" else make_orc_chain)(oracle, P[i], bq[i]) for i in range(N)]
    pos = bp.copy()
    for k, (frames, chunk) in enumerate(_chunks(pcm, CALLS, 6)):
        sub, pdm, st = eng.process_subframes_host(chunk, bd, frames)
        words, pdm2, st2 = twin.process_packets_host(chunk, bd, frames)
        assert sub.shape == (N, _pairs(flavour), sum(frames), 2, 2)
        for i in range(N):
            ws = _orc_words(oracle, flavour, chains[i], chunk[i], bd, frames)
            assert np.array_equal(words[i], ws), f"call {k} instance {i}: words differ from the oracle"
            assert np.array_equal(sub[i], oracle.spdif_encode(ws, int(pos[i]), bytes(cs[i]))), f"call {k} instance {i}: subframes"
        assert np.array_equal(sub, _two_pass(words, pos, cs)), f"call {k}: fused != two-pass"
        assert np.array_equal(pdm, pdm2) and st.tobytes() == st2.tobytes(), f"call {k}: PDM / status"
        pos = (pos + sum(frames)) % 192
        _check_tx(eng, pos, cs)
    assert np.any(st["clip_flags"] != 0), "no clipping exercised"


# ---- 2. position bookkeeping over words, subframe and output-less calls ----------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_every_call_advances_the_block_position(oracle, make_engine, flavour):
    N, fs, bd = 40, 48000.0, 16
    P, bq = _config(oracle, flavour, N, fs, 820)
    bp, cs = _tx(N, 821)
    calls = [CADENCE_44K1, [96, 96], [192, 1, 45], [44] * 3, [97, 95], [48] * 5]
    F_max = max(sum(c) for c in calls)
    pcm = pcm_bytes(N, sum(sum(c) for c in calls), bd, 822)
    eng, twin = make_engine(flavour, N, F_max), make_engine(flavour, N, F_max)
    for e in (eng, twin):
        _setup(e, P, bq)
    eng.set_spdif_tx(bp, cs)
    pos = bp.copy()
    d_pcm = torch.zeros(N * F_max * 4, dtype=torch.uint8, device="cuda")
    for k, (frames, chunk) in enumerate(_chunks(pcm, calls, 4)):
        words, _, _ = twin.process_packets_host(chunk, bd, frames)
        if k == 0:                                          # words form
            w, _, _ = eng.process_packets_host(chunk, bd, frames)
            assert np.array_equal(w, words)
        elif k == 1:                                        # a subframe call right after a words call continues the stream
            sub, _, _ = eng.process_subframes_host(chunk, bd, frames)
            assert np.array_equal(sub, _two_pass(words, pos, cs))
        elif k == 2:                                        # subframe form, every output NULL
            eng.process_subframes_host(chunk, bd, frames, want_subframes=False, want_pdm=False, want_status=False)
        elif k in (3, 4):                                   # device forms, every output NULL: words (3), subframes (4)
            d_pcm[:chunk.size] = torch.from_numpy(chunk.reshape(-1)).cuda()
            torch.cuda.synchronize()                        # the engine stream does not wait for torch's
            if k == 3:
                eng.process_packets_device(d_pcm.data_ptr(), bd, frames)
            else:
                eng.process_subframes_device(d_pcm.data_ptr(), bd, frames)
        else:                                               # and the stream is still continuous
            sub, _, _ = eng.process_subframes_host(chunk, bd, frames)
            assert np.array_equal(sub, _two_pass(words, pos, cs))
        pos = (pos + sum(frames)) % 192
        _check_tx(eng, pos, cs)


# ---- 3. the committed reference vectors --------------------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32s", "f32f", "q28"])
def test_reference_vectors_through_the_subframe_form(oracle, make_engine, flavour):
    """tests/golden/chain.npz (words of the reference's own compiled orchestrator) encoded by the oracle encoder"""
    g = load_golden("chain.npz")
    P, bq, pcm = g[f"{flavour}_params"], g[f"{flavour}_biquads"], np.ascontiguousarray(g[f"{flavour}_pcm"])
    npk, fpp = int(g["n_packets"]), int(g["fpp"])
    N = len(P)
    bp, cs = _tx(N, 830)
    eng = make_engine(flavour, N, npk * fpp)
    _setup(eng, P, bq)
    eng.set_spdif_tx(bp, cs)
    sub, pdm, status = eng.process_subframes_host(pcm, 24, [fpp] * npk)
    words = g[f"{flavour}_spdif"]
    for i in range(N):
        assert np.array_equal(sub[i], oracle.spdif_encode(words[i], int(bp[i]), bytes(cs[i]))), f"instance {i}"
    assert np.array_equal(pdm, g[f"{flavour}_pdm"])
    assert [int(s["clip_flags"]) for s in status] == [int(c) for c in g[f"{flavour}_clip"]]


# ---- 4. defaults, range setters and argument errors ----------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_defaults_ranges_and_errors(oracle, make_engine, flavour):
    N, fs, bd = 70, 48000.0, 24
    P, bq = _config(oracle, flavour, N, fs, 840)
    frames = [96, 96]
    pcm = pcm_bytes(N, sum(frames), bd, 841)
    eng, clean = make_engine(flavour, N, sum(frames)), make_engine(flavour, N, sum(frames))
    for e in (eng, clean):
        _setup(e, P, bq)
    cs = np.tile(np.frombuffer(DEFAULT_CS, np.uint8), (N, 1))
    bp = np.zeros(N, np.int64)
    _check_tx(eng, bp, cs)                                   # audio_spdif.c:82-88 bytes, position 0
    for e in (eng, clean):
        e.set_spdif_tx([5, 190], [[1, 2, 3, 4, 5], [6, 7, 8, 9, 10]], inst0=31)
        e.set_spdif_tx(191, bytes([0x04, 0, 0, 0x02, 0x0B]), inst0=69)
    bp[31:33], bp[69] = [5, 190], 191
    cs[31:33] = [[1, 2, 3, 4, 5], [6, 7, 8, 9, 10]]
    cs[69] = [0x04, 0, 0, 0x02, 0x0B]
    _check_tx(eng, bp, cs)
    got = eng.get_spdif_tx(2, inst0=31)
    assert list(got["block_pos"]) == [5, 190] and np.array_equal(got["reserved"], np.zeros((2, 2), np.uint8))

    lib = api.lib()
    pre = "dspi_chainq" if flavour == "q28" else "dspi_chain"
    set_, get_ = getattr(lib, pre + "_set_spdif_tx"), getattr(lib, pre + "_get_spdif_tx")
    rec = np.zeros(3, L.SPDIF_TX)
    rec["block_pos"] = [7, 8, 9]
    rec["channel_status"] = [9, 9, 9, 9, 9]
    p = rec.ctypes.data_as(C.c_void_p)
    assert set_(eng._h, 69, 2, p) == -34                    # one past the end
    assert set_(eng._h, 71, 0, p) == -34                    # start past the end
    assert set_(eng._h, 0xFFFFFFFF, 2, p) == -34            # end wraps in 32 bits
    assert get_(eng._h, 0xFFFFFFFF, 2, p) == -34
    assert get_(eng._h, 60, 11, p) == -34
    assert set_(eng._h, 0, 1, None) == -22
    assert get_(eng._h, 0, 1, None) == -22
    assert set_(None, 0, 1, p) == -22
    rec["block_pos"][2] = 192                               # one bad record: nothing written
    assert set_(eng._h, 10, 3, p) == -22
    assert set_(eng._h, 10, 0, p) == 0                      # n = 0: no-op
    assert get_(eng._h, 70, 0, p) == 0
    with pytest.raises(api.DspiError):
        eng.set_spdif_tx(300, DEFAULT_CS, inst0=0)
    _check_tx(eng, bp, cs)
    a = eng.process_subframes_host(pcm, bd, frames)
    b = clean.process_subframes_host(pcm, bd, frames)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    _check_tx(eng, bp + sum(frames), cs)


# ---- 5. checkpoint: state blob + transmitter state ---------------------------------------------------------------------------
@pytest.mark.parametrize("flavour,cpl,cpl_resume", [("f32f", "1", "2"), ("f32s", "2", "1"), ("q28", None, None)], ids=["f32f", "f32s", "q28"])
def test_checkpoint_resumes_the_stream(libm_f64, make_engine, flavour, cpl, cpl_resume):
    oracle = libm_f64
    N, fs, bd = 70, 48000.0, 24
    P, bq = _config(oracle, flavour, N, fs, 850)
    bp, cs = _tx(N, 851)
    calls = CALLS[:2]
    F_max = max(sum(c) for c in calls)
    pcm = pcm_bytes(N, sum(sum(c) for c in calls), bd, 852)
    run, plain = make_engine(flavour, N, F_max, cpl), make_engine(flavour, N, F_max, cpl)
    for e in (run, plain):
        _setup(e, P, bq)
    run.set_spdif_tx(bp, cs)
    parts = list(_chunks(pcm, calls, 6))
    run.process_subframes_host(parts[0][1], bd, parts[0][0])
    plain.process_subframes_host(parts[0][1], bd, parts[0][0])
    blob, tx = run.state_export(), run.get_spdif_tx()
    # the transmitter state is not in the blob: an engine at other positions exports the same bytes
    assert np.array_equal(blob, plain.state_export())
    assert int(np.frombuffer(blob[:8].tobytes(), np.uint32)[1]) == (1 if flavour == "q28" else 2)
    assert int(np.frombuffer(blob[24:32].tobytes(), np.uint64)[0]) == blob.size
    resumed = make_engine(flavour, N, F_max, cpl_resume)
    _setup(resumed, P, bq)
    resumed.state_import(blob)
    resumed.set_spdif_tx(tx["block_pos"], tx["channel_status"])
    a = run.process_subframes_host(parts[1][1], bd, parts[1][0])
    b = resumed.process_subframes_host(parts[1][1], bd, parts[1][0])
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    _check_tx(resumed, bp + sum(calls[0]) + sum(calls[1]), cs)


# ---- 6. reset_state keeps the transmitter state ----------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32s", "q28"])
def test_reset_state_keeps_the_transmitter(oracle, make_engine, flavour):
    N, fs, bd = 33, 48000.0, 16
    P, bq = _config(oracle, flavour, N, fs, 860)
    bp, cs = _tx(N, 861)
    eng = make_engine(flavour, N, 441)
    _setup(eng, P, bq)
    eng.set_spdif_tx(bp, cs)
    eng.process_subframes_host(pcm_bytes(N, 441, bd, 862), bd, CADENCE_44K1)
    before = eng.get_spdif_tx()
    eng.reset_state()
    assert before.tobytes() == eng.get_spdif_tx().tobytes()
    _check_tx(eng, bp + 441, cs)


# ---- 7. a setter right behind an asynchronous call --------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_setter_is_ordered_behind_an_asynchronous_call(oracle, make_engine, flavour):
    N, fs, bd = 2048, 96000.0, 24
    P, bq = (W.chain_config3_q28(N, fs=fs) if flavour == "q28" else W.chain_config3(N, fs=fs, seed=3))
    frames = [96] * 16
    F = sum(frames)
    bp, cs = _tx(N, 871)
    eng, twin = make_engine(flavour, N, F), make_engine(flavour, N, F)
    for e in (eng, twin):
        _setup(e, P, bq)
    eng.set_spdif_tx(bp, cs)
    pcm = [pcm_bytes(N, F, bd, 872 + k) for k in range(2)]
    pairs = _pairs(flavour)
    d_pcm = torch.from_numpy(pcm[0]).cuda()
    d_sub = torch.empty((N, pairs, F, 2, 2), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    eng.process_subframes_device(d_pcm.data_ptr(), bd, frames, d_sub.data_ptr())
    new_bp = (bp * 7 + 3) % 192
    new_cs = cs.copy()
    new_cs[:, 3] ^= 0x0F
    eng.set_spdif_tx(new_bp, new_cs)                        # issued while the call may still run
    eng.sync()
    first = d_sub.cpu().numpy().view(np.uint32)
    w0, _, _ = twin.process_packets_host(pcm[0], bd, frames)
    assert np.array_equal(first, _two_pass(w0, bp, cs)), "the setter changed the call before it"
    w1, _, _ = twin.process_packets_host(pcm[1], bd, frames)
    sub1, _, _ = eng.process_subframes_host(pcm[1], bd, frames)
    assert np.array_equal(sub1, _two_pass(w1, new_bp, new_cs)), "the setter did not apply to the next call"


# ---- 8. host form, device form and the two-pass path at scale ---------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "q28"])
def test_host_device_and_two_pass_agree_at_scale(make_engine, flavour):
    N, fs, bd = 8192, 96000.0, 24
    P, bq = (W.chain_config3_q28(N, fs=fs) if flavour == "q28" else W.chain_config3(N, fs=fs, seed=1))
    frames = [96, 96]
    F, pairs = sum(frames), _pairs(flavour)
    # six (position, status) classes, so that the two-pass reference is six whole-buffer encoder runs
    variants = [(bpv, csv) for bpv in (0, 1, 191) for csv in (DEFAULT_CS, bytes([0x04, 0, 0, 0x0E, 0x0B]))]
    cls = np.arange(N) % len(variants)
    bp = np.array([variants[c][0] for c in cls])
    cs = np.stack([np.frombuffer(variants[c][1], np.uint8) for c in cls])
    host, dev, words = (make_engine(flavour, N, F) for _ in range(3))
    for e in (host, dev, words):
        _setup(e, P, bq)
    host.set_spdif_tx(bp, cs)
    dev.set_spdif_tx(bp, cs)
    pcm = torch.randint(0, 256, (N, F * 6), dtype=torch.uint8, device="cuda")
    for call in range(2):
        pcm.random_(0, 256)
        h_sub, h_pdm, h_st = host.process_subframes_host(pcm.cpu().numpy(), bd, frames)
        d_sub = torch.empty((N, pairs, F, 2, 2), dtype=torch.int32, device="cuda")
        d_pdm = torch.zeros((N, F, 8), dtype=torch.int32, device="cuda")
        d_st = torch.zeros((N * h_st.dtype.itemsize,), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        dev.process_subframes_device(pcm.data_ptr(), bd, frames, d_sub.data_ptr(), d_pdm.data_ptr(), d_st.data_ptr())
        d_words = torch.empty((N, pairs, F, 2), dtype=torch.int32, device="cuda")
        words.process_packets_device(pcm.data_ptr(), bd, frames, d_words.data_ptr())
        words.sync()
        dev.sync()
        want = torch.empty_like(d_sub)
        tmp = torch.empty_like(d_sub)
        for c, (bpv, csv) in enumerate(variants):
            api.spdif_encode_device(d_words.data_ptr(), N * pairs, F, tmp.data_ptr(), block_pos0=(bpv + call * F) % 192, channel_status=csv)
            torch.cuda.synchronize()
            sel = torch.from_numpy(cls == c).cuda()
            want[sel] = tmp[sel]
        assert torch.equal(d_sub, want), f"call {call}: fused != two-pass"
        assert np.array_equal(h_sub, d_sub.cpu().numpy().view(np.uint32)), f"call {call}: host != device"
        assert np.array_equal(h_pdm, d_pdm.cpu().numpy().view(np.uint32)) and h_st.tobytes() == d_st.cpu().numpy().tobytes()
