"""K1 (float cascade) and K2 (Q28 cascade) against the oracle across their configurations, output words and downloaded
filter state bit for bit.

K1 is instantiated for 10 and for 12 bands, in two stage geometries (one channel per lane with 32 x 64 stages, the
default; a register pair per lane with 64 x 32 stages, DSPI_F32_CPL=2), in two arithmetic flavours, and takes one of
several paths per warp: the straight-line register-tile path (all-biquad warps), the band-outer column path, the
run-time specialised kernel (DSPI_JIT=force) and the dynamic time-slice schedule (DSPI_DBG=8).  K2 has template
instances for 10 and 12 bands at register tiles of 8 or 4 samples (DSPI_K2_SUB) and a per-band branch path
(DSPI_K2_PLAIN=0).  Every case checks which kernel the engine reports, so that a case cannot silently run another
path than the one it is about.

Every float batch mixes seeded noise, an impulse, a silent channel, channels of subnormal samples and channels whose
uploaded records carry subnormal filter state: the firmware runs with flush-to-zero and denormals-are-zero, so a
subnormal operand counts as zero on every path.

Range calls (dspi_eq_process_device_range) whose channel count is not a multiple of the group size must leave every
channel outside the range untouched, state included.  Chain checkpoints must resume in an engine created under the
other K1 geometry."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L, workloads as W                     # noqa: E402
from tests.chain_cases import chain_params, pcm_bytes                        # noqa: E402
from tests.util import same_bits                                             # noqa: E402

FS = 96000.0
GEOMETRY = {1: "tile 32 rows x 64 samples", 2: "tile 64 rows x 32 samples"}
C_F = 100                                   # a partial last group in either geometry (32 or 64 rows)
T_F = 295                                   # 4 whole 64-sample stages + a 39-sample tail: one 32-sample box and a ragged 7
SPLITS = [96, 199]                          # 64 + 32 (the tail stays straight-line), then 3 stages + 7
SUBNORMAL_STATE_ROWS = [7, 20, 21, 22, 23, C_F - 1]


def _subnormals(rng, shape):
    """float32 subnormals of both signs: raw bit patterns 1..0x007FFFFF, random sign bit"""
    bits = rng.integers(1, 0x00800000, shape, dtype=np.uint32) | (rng.integers(0, 2, shape, dtype=np.uint32) << np.uint32(31))
    return bits.view(np.float32)


def _float_inputs(Cn, T, seed=1):
    rng = np.random.default_rng(seed)
    x = W.inputs_f32(Cn, T)
    x[3] = 0
    x[3, 0] = 1.0                                               # impulse: decays into the flush-to-zero range
    x[7] = 0                                                    # silence (its records carry subnormal state)
    x[11] = _subnormals(rng, T)
    x[12] = _subnormals(rng, T)
    x[13, 1::2] = _subnormals(rng, x[13, 1::2].shape)           # noise interleaved with subnormals
    return x


def _with_subnormal_state(bq, rows, seed=2):
    """records of `rows` carry subnormal state in every band (TDF2 s1/s2 and SVF ic1eq/ic2eq): it must flush on first use"""
    rng = np.random.default_rng(seed)
    for f in ("s1", "s2", "svic1eq", "svic2eq"):
        bq[f][rows] = _subnormals(rng, (len(rows), L.MAX_BANDS))
    return bq


def _float_coeffs(variant, Cn, n_bands, seed=5):
    bq = api.compute_coefficients(W.eq_params(variant, Cn, fs=FS, nbands=n_bands, seed=seed), q28=False, fs=FS)
    return _with_subnormal_state(bq, [r for r in SUBNORMAL_STATE_ROWS if r < Cn])


def _oracle(oracle, flavour, bq, x, n_bands):
    b, y = bq.copy(), x.copy()
    oracle.eq_many(flavour, b, y, n_bands, 96)
    return y, b


def _run(monkeypatch, cpl, flavour, bq, x, n_bands, splits=None, ld=None):
    """x [C, T] through a fresh engine created under DSPI_F32_CPL=cpl; rows padded to a multiple of 4 floats (TMA path)
    unless `ld` says otherwise.  Returns (y, final biquads, kernel info)."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    Cn, T = x.shape
    ld = (T + 3) // 4 * 4 if ld is None else ld
    eng = api.EqEngine(flavour, Cn, n_bands)
    try:
        eng.upload(bq)
        info = eng.kernel_info()
        buf = torch.zeros((Cn, ld), dtype=torch.float32, device="cuda")
        buf[:, :T] = torch.from_numpy(x).cuda()
        torch.cuda.synchronize()
        t0 = 0
        for n in (splits or [T]):
            eng.process_device(buf.data_ptr() + t0 * 4, n, ld)
            t0 += n
        eng.sync()
        return buf[:, :T].cpu().numpy(), eng.download(), info
    finally:
        eng.close()


def _check(oracle, monkeypatch, cpl, flavour, bq, x, n_bands, splits=None, ld=None):
    """one engine against the same-flavour oracle; returns the kernel info after checking the geometry it names"""
    want, wst = _oracle(oracle, flavour, bq, x, n_bands)
    y, st, info = _run(monkeypatch, cpl, flavour, bq, x, n_bands, splits=splits, ld=ld)
    assert GEOMETRY[cpl] in info, info
    bad = np.argwhere(y.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, (f"{info}: {len(bad)} samples differ from the oracle, first at channel {bad[0][0]} sample {bad[0][1]}: "
                           f"gpu {y[tuple(bad[0])]!r} oracle {want[tuple(bad[0])]!r}")
    assert same_bits(st, wst), f"{info}: filter state differs from the oracle in channels " \
                               f"{sorted(set(np.argwhere(st != wst)[:, 0].tolist()))[:16]}"
    return info


def _svf_zero_sign(request):
    """Known deviation, kept visible: svf_tile() (register tiles and column path) keeps the SVF state negated on alternate
    samples, and an exactly cancelling sum rounds to +0 whichever operand is negated.  Where the reference's output is
    -0.0 (a channel of negative subnormals, flushed to -0.0, through a single shelving SVF band) K1 gives +0.0; a later
    band maps both zeros to the same value, so only one-band engines show it.  Strict: the case fails once it passes."""
    request.applymarker(pytest.mark.xfail(strict=True, reason="SVF register tiles give +0.0 where the reference gives -0.0"))


def _aot_path(variant, n_bands):
    """the ahead-of-time path an engine of fewer than 1024 channels reports: all-biquad warps at the kernel's own band
    count (10 or 12) run straight-line, everything else the column path"""
    return "aot straight-line biquad" if variant == "A" and n_bands in (10, 12) else "aot generic column path"


# ---- K1: band counts x geometry x flavour x topology --------------------------------------------------------------
@pytest.mark.parametrize("variant", ["A", "B", "mixed"])
@pytest.mark.parametrize("flavour", ["f32f", "f32s"])
@pytest.mark.parametrize("cpl", [1, 2])
@pytest.mark.parametrize("n_bands", [1, 2, 9, 10, 11, 12])
def test_float_band_counts(request, monkeypatch, oracle, n_bands, cpl, flavour, variant):
    """n_bands 1..10 run the 10-band instances with the bands >= n masked off, 11 and 12 the 12-band instances; one
    launch of 295 samples, and the same in two launches so that state carries between calls"""
    if variant == "B" and n_bands == 1:
        _svf_zero_sign(request)
    monkeypatch.delenv("DSPI_JIT", raising=False)
    monkeypatch.delenv("DSPI_DBG", raising=False)
    bq = _float_coeffs(variant, C_F, n_bands)
    x = _float_inputs(C_F, T_F)
    info = _check(oracle, monkeypatch, cpl, flavour, bq, x, n_bands)
    assert info.startswith(_aot_path(variant, n_bands)), info
    _check(oracle, monkeypatch, cpl, flavour, bq, x, n_bands, splits=SPLITS)


# ---- K1: forced paths on a subset of band counts --------------------------------------------------------------------
FORCED_BANDS = [1, 9, 11, 12]


def _alt_flavour(n_bands, cpl):
    return "f32f" if (n_bands + cpl) % 2 else "f32s"


@pytest.mark.parametrize("cpl", [1, 2])
@pytest.mark.parametrize("n_bands", FORCED_BANDS)
def test_float_specialised_kernel_band_counts(request, monkeypatch, oracle, n_bands, cpl):
    """DSPI_JIT=force: the kernel is compiled for the dominant topology vector of n bands (bands >= n are bypass in the
    signature); a block of channels of other topologies takes the generic path inside the same kernel.  One flavour per
    (band count, geometry) pair, alternating, keeps the number of run-time compilations down."""
    monkeypatch.setenv("DSPI_JIT", "force")
    monkeypatch.delenv("DSPI_DBG", raising=False)
    flavour = _alt_flavour(n_bands, cpl)
    if n_bands == 1 and cpl == 1:                                   # the (1 band, 2 ch/lane) case ends with the reference's zeros
        _svf_zero_sign(request)
    bq = _float_coeffs("B", C_F, n_bands)
    other = _float_coeffs("mixed", C_F, n_bands, seed=11)
    for c in range(40, 46):
        bq[c] = other[c]
    x = _float_inputs(C_F, T_F)
    info = _check(oracle, monkeypatch, cpl, flavour, bq, x, n_bands)
    assert info.startswith("jit sig=0x"), info
    sig = int(info.split()[1][len("sig="):], 16)
    assert sig != 0 and sig >> (4 * n_bands) == 0, f"signature must bypass bands >= {n_bands}: {info}"
    assert f"nb={10 if n_bands <= 10 else 12} " in info, info
    _check(oracle, monkeypatch, cpl, flavour, bq, x, n_bands, splits=SPLITS)


@pytest.mark.parametrize("variant", ["A", "mixed"])
@pytest.mark.parametrize("cpl", [1, 2])
@pytest.mark.parametrize("n_bands", FORCED_BANDS)
def test_float_column_path_band_counts(monkeypatch, oracle, n_bands, cpl, variant):
    """DSPI_DBG=4 sends every warp down the column path, the all-biquad ones included"""
    monkeypatch.delenv("DSPI_JIT", raising=False)
    monkeypatch.setenv("DSPI_DBG", "4")
    flavour = _alt_flavour(n_bands, cpl)
    bq = _float_coeffs(variant, C_F, n_bands)
    x = _float_inputs(C_F, T_F)
    info = _check(oracle, monkeypatch, cpl, flavour, bq, x, n_bands)
    assert info.startswith(_aot_path(variant, n_bands)), info
    _check(oracle, monkeypatch, cpl, flavour, bq, x, n_bands, splits=SPLITS)


@pytest.mark.parametrize("variant", ["A", "mixed"])
@pytest.mark.parametrize("cpl", [1, 2])
@pytest.mark.parametrize("n_bands", FORCED_BANDS)
def test_float_dynamic_schedule_band_counts(monkeypatch, oracle, n_bands, cpl, variant):
    """DSPI_DBG=8 (T >= 1024, rows a multiple of 4 floats): a persistent grid pulls (group, 512-sample slice) items and
    the filter state travels between slices through the coefficient store; strict flavour, all-biquad warps on the
    straight-line path and mixed-topology warps on the column path"""
    monkeypatch.delenv("DSPI_JIT", raising=False)
    monkeypatch.setenv("DSPI_DBG", "8")
    T = 2048 + 40
    bq = _float_coeffs(variant, C_F, n_bands, seed=14)
    x = _float_inputs(C_F, T)
    info = _check(oracle, monkeypatch, cpl, "f32s", bq, x, n_bands)
    assert info.startswith(_aot_path(variant, n_bands)), info
    _check(oracle, monkeypatch, cpl, "f32s", bq, x, n_bands, splits=[1024 + 64, T - 1024 - 64])


# ---- K2: band counts x bypass shapes, and its two static switches ---------------------------------------------------
Q28_BANDS = [1, 7, 10, 11, 12]
Q28_SHAPES = ["all_on", "mixed", "one_band_flat_everywhere"]


def q28_case(oracle, n_bands, shape):
    """100 channels (a partial last warp) x 1000 samples in two launches, a wrap-around channel; bit-exact output and state"""
    fs, Cn, T = 48000.0, 100, 1000
    params = W.eq_params("mixed" if shape == "mixed" else "A", Cn, fs=fs, nbands=n_bands, seed=21)
    if shape == "one_band_flat_everywhere":
        params["gain_db"][:, n_bands // 2] = 0.0
        params["type"][:, n_bands // 2] = L.PEAKING
    bq = api.compute_coefficients(params, q28=True, fs=fs)
    if shape == "all_on":
        assert not bq["bypass"][:, :n_bands].any()
    if shape == "one_band_flat_everywhere":
        assert bq["bypass"][:, n_bands // 2].all()
    rng = np.random.default_rng(n_bands)
    bq["s1"] = rng.integers(-2**27, 2**27, bq.shape, dtype=np.int64).astype(np.int32)      # live state on entry
    bq["s2"] = rng.integers(-2**27, 2**27, bq.shape, dtype=np.int64).astype(np.int32)
    x = W.inputs_q28(Cn, T)
    x[5] = np.random.default_rng(3).integers(-2**31, 2**31, T, dtype=np.int64).astype(np.int32)          # wrap-around stress
    x[9] = 0
    eng = api.EqEngine("q28", Cn, n_bands)
    try:
        eng.upload(bq)
        info = eng.kernel_info()
        buf = torch.from_numpy(x).cuda()
        eng.process_device(buf.data_ptr(), 504, T)
        eng.process_device(buf.data_ptr() + 504 * 4, T - 504, T)
        eng.sync()
        y, st = buf.cpu().numpy(), eng.download()
    finally:
        eng.close()
    assert info.startswith("aot q28 cascade"), info
    want, wst = x.copy(), bq.copy()
    oracle.eq_many("q28", wst, want, n_bands, 96)
    assert np.array_equal(y, want), f"q28 n_bands={n_bands} {shape}: samples differ"
    assert same_bits(st, wst), f"q28 n_bands={n_bands} {shape}: filter state differs"


@pytest.mark.parametrize("shape", Q28_SHAPES)
@pytest.mark.parametrize("n_bands", Q28_BANDS)
def test_q28_band_counts(oracle, n_bands, shape):
    q28_case(oracle, n_bands, shape)


@pytest.mark.parametrize("env", [{"DSPI_K2_SUB": "4"}, {"DSPI_K2_PLAIN": "0"}], ids=["sub4", "plain0"])
def test_q28_switches(oracle, env):
    """DSPI_K2_SUB=4 selects the 4-sample register-tile instances, DSPI_K2_PLAIN=0 the per-band branch path for every
    warp.  Both are read once per process, so the whole Q28 set runs in a subprocess."""
    code = textwrap.dedent(f'''
        from tests.orc import Oracle
        from tests.test_eq_matrix_gpu import q28_case
        orc = Oracle()
        for n in {Q28_BANDS!r}:
            for shape in {Q28_SHAPES!r}:
                q28_case(orc, n, shape)
        print("ok")
    ''')
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=600,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr


# ---- range calls: channels outside the range keep their samples and their state ------------------------------------
RANGE_C = 300


def _range_ranges(Cn):
    return [(0, Cn), (0, 40), (64, 70), (192, Cn - 192 - 7), (0, Cn)]


@pytest.mark.parametrize("arith,cpl,mode", [("f32f", 1, "tma"), ("f32f", 2, "tma"), ("f32s", 1, "plain"), ("f32f", 2, "plain"),
                                            ("f32f", 1, "dynamic"), ("f32s", 2, "dynamic"), ("q28", 1, "tma"), ("q28", 1, "plain")])
def test_range_calls_leave_other_channels_untouched(monkeypatch, oracle, arith, cpl, mode):
    """After a whole call has given every channel live state, range calls whose channel count is not a multiple of the
    group ((0, 40), (64, 70), (192, 101) of 300 channels) process their channels exactly like the oracle run on those
    channels alone, and leave every other channel's samples and filter state byte for byte as they were; a final whole
    call shows that the neighbours of each range carry on from their own state.  `plain`: a row stride that is not a
    multiple of 4 elements (plain loads and stores); `dynamic`: DSPI_DBG=8."""
    monkeypatch.delenv("DSPI_JIT", raising=False)
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    if mode == "dynamic":
        monkeypatch.setenv("DSPI_DBG", "8")
    else:
        monkeypatch.delenv("DSPI_DBG", raising=False)
    q28 = arith == "q28"
    Cn, nb = RANGE_C, 10
    T = 1088 if mode == "dynamic" else 295
    ld = T + 3 if mode == "plain" else (T + 3) // 4 * 4
    if mode == "plain":
        assert ld % 4 != 0
    variant = "mixed" if arith != "f32f" else "B"
    params = W.eq_params(variant, Cn, fs=FS, nbands=nb, seed=31)
    bq = api.compute_coefficients(params, q28=q28, fs=FS)
    dt = np.int32 if q28 else np.float32

    def inputs(k):
        return W.inputs_q28(Cn, T, ch0=4096 * k) if q28 else W.inputs_f32(Cn, T, ch0=4096 * k)

    eng = api.EqEngine(arith, Cn, nb)
    try:
        eng.upload(bq)
        if not q28:
            assert GEOMETRY[cpl] in eng.kernel_info()
        ost = bq.copy()                                          # the oracle's state of every channel
        for k, (a, n) in enumerate(_range_ranges(Cn)):
            x = inputs(k)
            host = np.zeros((Cn, ld), dt)
            host[:, :T] = x
            buf = torch.from_numpy(host).cuda()
            before = eng.download()
            torch.cuda.synchronize()
            if (a, n) == (0, Cn):
                eng.process_device(buf.data_ptr(), T, ld)
            else:
                eng.process_device_range(buf[a].data_ptr(), T, ld, a, n)
            eng.sync()
            y, st = buf.cpu().numpy()[:, :T], eng.download()
            want, wst = x[a:a + n].copy(), ost[a:a + n].copy()
            oracle.eq_many(arith, wst, want, nb, 96)
            ost[a:a + n] = wst
            out = np.r_[0:a, a + n:Cn]
            assert np.array_equal(y[a:a + n].view(np.uint32), want.view(np.uint32)), f"range ({a}, {n}): samples differ from the oracle"
            assert same_bits(st[a:a + n], wst), f"range ({a}, {n}): filter state differs from the oracle"
            assert np.array_equal(y[out].view(np.uint32), x[out].view(np.uint32)), f"range ({a}, {n}): samples outside the range changed"
            changed = sorted(set(np.argwhere(st[out] != before[out])[:, 0].tolist()))
            assert same_bits(st[out], before[out]), \
                f"range ({a}, {n}): filter state of channels outside the range changed: {[int(out[i]) for i in changed][:12]}"
            assert same_bits(st, ost)
    finally:
        eng.close()


# ---- chain checkpoints across K1 geometries -------------------------------------------------------------------------
def _chain_run(monkeypatch, cpl, N, P, bq, pcms, blob=None, export_after=None):
    """a float chain engine created under DSPI_F32_CPL=cpl: optionally import `blob`, then process each of `pcms`;
    returns the outputs of every call, the final biquads and (after call `export_after`) an exported blob"""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    npk, fpp, bits = 3, 96, 24
    e = api.ChainEngine("f32f", N, max_frames=npk * fpp)
    try:
        e.set_params(P)
        e.upload_biquads(bq)
        if blob is not None:
            e.state_import(blob)
        outs, exported = [], None
        for i, pcm in enumerate(pcms):
            spdif, pdm, status = e.process_host(pcm, bits, npk, fpp)
            outs.append((spdif.copy(), pdm.copy(), status.copy()))
            if i == export_after:
                exported = e.state_export()
        return outs, e.download_biquads(), exported
    finally:
        e.close()


def _v1_blob(blob):
    """the same checkpoint in the version 1 layout: a 32-byte header without the geometry fields"""
    b = np.asarray(blob, np.uint8)
    hdr = b[:40].copy()
    assert hdr[:8].view(np.uint32)[1] == 2 and tuple(hdr[32:40].view(np.uint32)) == (1, 1)
    hdr[4:8] = np.array([1], np.uint32).view(np.uint8)
    hdr[24:32] = np.array([b.size - 8], np.uint64).view(np.uint8)
    return np.concatenate([hdr[:32], b[40:]])


@pytest.mark.parametrize("N", [64, 20])
@pytest.mark.parametrize("src,dst", [(1, 2), (2, 1)])
def test_chain_checkpoint_across_geometries(monkeypatch, oracle, N, src, dst):
    """a checkpoint exported under one K1 geometry resumes in an engine created under the other one: same S/PDIF words,
    PDM words, status and filter state as the uninterrupted run.  N = 64 gives both geometries the same byte count,
    N = 20 (32 padded instances, 288 output rows) a different one."""
    monkeypatch.delenv("DSPI_DBG", raising=False)
    P, bq = chain_params(oracle, N, FS, 41)
    pcms = [pcm_bytes(N, 3 * 96, 24, s) for s in (1, 2, 3)]
    want, wst, blob = _chain_run(monkeypatch, src, N, P, bq, pcms, export_after=0)

    def resume(b):
        got, gst, _ = _chain_run(monkeypatch, dst, N, P, bq, pcms[1:], blob=b)
        for call, ((s1, p1, t1), (s2, p2, t2)) in enumerate(zip(want[1:], got)):
            assert np.array_equal(s1, s2), f"call {call}: S/PDIF words differ after resuming under the other geometry"
            assert np.array_equal(p1, p2), f"call {call}: PDM words differ after resuming under the other geometry"
            assert t1.tobytes() == t2.tobytes(), f"call {call}: status differs after resuming under the other geometry"
        assert same_bits(gst, wst), "filter state differs after resuming under the other geometry"
    resume(blob)
    if src == 1:
        resume(_v1_blob(blob))                                      # version 1 blobs are read as one channel per lane
    assert not np.array_equal(want[1][0], 0 * want[1][0])
