"""K1's two stage geometries against the oracle and against each other, output and filter state bit for bit.

One channel per lane with stages of 32 rows x 64 samples is the default; a register pair per lane with stages of
64 rows x 32 samples is selected with DSPI_F32_CPL=2 when an engine is created.  The cases are the shapes on which
the two geometries take different paths: tails that are not whole 64-sample stages, strides that force the
plain-load path, the column path, the run-time specialised kernel, launches whose lengths alternate between
multiples of 32 and 64 samples, and the chain engine's packet slices."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, workloads as W                                   # noqa: E402
from tests.chain_cases import chain_params, pcm_bytes                        # noqa: E402
from tests.util import same_bits                                             # noqa: E402

FS = 96000.0
GEOMETRY = {1: "tile 32 rows x 64 samples", 2: "tile 64 rows x 32 samples"}


def _coeffs(variant, Cn, seed=5):
    return api.compute_coefficients(W.eq_params(variant, Cn, fs=FS, seed=seed), q28=False, fs=FS)


def _run(monkeypatch, cpl, flavour, bq, x, splits=None, ld=None, n_bands=10):
    """x [C, T] through a fresh engine of `cpl` channels per lane; returns (y, final biquads, kernel info)."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    Cn, T = x.shape
    ld = T if ld is None else ld
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


def _both(monkeypatch, oracle, flavour, bq, x, n_bands=10, **kw):
    """runs both geometries, checks each against the oracle and the two against each other; returns the two infos"""
    want, wst = x.copy(), bq.copy()
    oracle.eq_many(flavour, wst, want, n_bands, 96)
    out = {}
    for cpl in (1, 2):
        y, st, info = _run(monkeypatch, cpl, flavour, bq, x, n_bands=n_bands, **kw)
        assert GEOMETRY[cpl] in info, info
        assert np.array_equal(y.view(np.uint32), want.view(np.uint32)), f"cpl={cpl}: samples differ from the oracle ({info})"
        assert same_bits(st, wst), f"cpl={cpl}: filter state differs from the oracle ({info})"
        out[cpl] = (y, st, info)
    assert np.array_equal(out[1][0].view(np.uint32), out[2][0].view(np.uint32))
    assert same_bits(out[1][1], out[2][1])
    return out[1][2], out[2][2]


@pytest.mark.parametrize("variant", ["A", "mixed"])
@pytest.mark.parametrize("T", [96, 33, 6144 + 40])
def test_tails_not_a_multiple_of_the_stage(monkeypatch, oracle, variant, T):
    """96 = 64 + 32 keeps the straight-line path for its 32-sample tail; 33 and 6184 leave ragged tails (a stage whose
    second 32-sample box starts past the end of the row for 33 + 31 of its 64 samples)"""
    Cn = 100                                                     # a partial last group in either geometry
    bq = _coeffs(variant, Cn)
    x = W.inputs_f32(Cn, T)
    x[3] = 0
    x[3, 0] = 1.0
    _both(monkeypatch, oracle, "f32f", bq, x)


@pytest.mark.parametrize("variant", ["A", "mixed"])
def test_padded_stride_takes_the_plain_load_path(monkeypatch, oracle, variant):
    """a row stride that is not a multiple of 4 floats cannot be described to the TMA unit: plain loads and stores
    through the same stage layout"""
    Cn, T = 70, 200
    _both(monkeypatch, oracle, "f32s", _coeffs(variant, Cn, seed=8), W.inputs_f32(Cn, T), ld=T + 3)


@pytest.mark.parametrize("variant", ["A", "mixed"])
def test_column_path(monkeypatch, oracle, variant):
    """DSPI_DBG=4 sends every warp down the band-outer column path, which re-lays the stage out as lane columns"""
    monkeypatch.setenv("DSPI_DBG", "4")
    Cn, T = 130, 1000
    _both(monkeypatch, oracle, "f32f", _coeffs(variant, Cn, seed=12), W.inputs_f32(Cn, T))


def test_dynamic_time_slice_schedule(monkeypatch, oracle):
    """DSPI_DBG=8: a persistent grid pulls (group, 512-sample slice) items; filter state travels between slices"""
    monkeypatch.setenv("DSPI_DBG", "8")
    Cn, T = 300, 2048 + 40
    _both(monkeypatch, oracle, "f32f", _coeffs("A", Cn, seed=14), W.inputs_f32(Cn, T))


@pytest.mark.parametrize("flavour", ["f32f", "f32s"])
def test_specialised_kernel(monkeypatch, oracle, flavour):
    """the NVRTC kernel is compiled for the engine's geometry; 200 channels x 100 samples end in ragged group and tile"""
    monkeypatch.setenv("DSPI_JIT", "force")
    Cn, T = 200, 100
    info1, info2 = _both(monkeypatch, oracle, flavour, _coeffs("B", Cn), W.inputs_f32(Cn, T))
    assert info1.startswith("jit sig=0x") and info2.startswith("jit sig=0x"), (info1, info2)


@pytest.mark.parametrize("variant", ["A", "B"])
def test_state_across_calls_of_32_and_64_multiples(monkeypatch, oracle, variant):
    """launch lengths alternate between multiples of 32 and of 64 samples (and one of neither)"""
    splits = [64, 32, 96, 64, 32, 128, 40, 24]
    Cn = 96
    x = W.inputs_f32(Cn, sum(splits))
    _both(monkeypatch, oracle, "f32f", _coeffs(variant, Cn, seed=3), x, splits=splits)


@pytest.mark.parametrize("fpp,n_packets", [(96, 6), (45, 7)])
def test_chain_engine_same_bits_in_both_geometries(monkeypatch, oracle, fpp, n_packets):
    """the chain engines run K1 over slices of whole packets: 96-frame packets give 64 + 32-sample stages, 45-frame
    packets slices that start off 16-byte boundaries (plain-load path)"""
    N = 40
    P, bq = chain_params(oracle, N, FS, 31)
    pcm = pcm_bytes(N, fpp * n_packets * 2, 24, 32)
    half = pcm.shape[1] // 2
    got = {}
    for cpl in (1, 2):
        monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
        eng = api.ChainEngine("f32f", N, max_frames=fpp * n_packets)
        try:
            eng.set_params(P)
            eng.upload_biquads(bq)
            outs = []
            for call in range(2):                               # state carried across calls
                spdif, pdm, status = eng.process_host(np.ascontiguousarray(pcm[:, call * half:(call + 1) * half]), 24, n_packets, fpp)
                outs.append((spdif.copy(), pdm.copy(), status.copy()))
            got[cpl] = (outs, eng.download_biquads())
        finally:
            eng.close()
    for (s1, p1, st1), (s2, p2, st2) in zip(got[1][0], got[2][0]):
        assert np.array_equal(s1, s2), "S/PDIF words differ between geometries"
        assert np.array_equal(p1, p2), "PDM bits differ between geometries"
        assert same_bits(st1, st2), "status differs between geometries"
    assert same_bits(got[1][1], got[2][1]), "filter state differs between geometries"
