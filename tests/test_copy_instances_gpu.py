"""GPU: dspi_chain(q)_copy_instances - instances copied between slots of one engine on the device.
The bar is a twin engine, driven identically, that moves the same pairs the host way: export_instances(src[k], 1) then
import_instances(dst[k], 1) per pair.  Both engines must then hold the same bytes (whole-engine instance images and state
blob) and give the same outputs on later calls; copied instances also continue against the oracle chains of their
sources.  Float engines run both K1 geometries (DSPI_F32_CPL 1 and 2), so 64-row EQ groups are shared with
non-destinations in either."""
import ctypes as C
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                                  # noqa: E402
from tests.chain_cases import pcm_bytes                                                  # noqa: E402
from tests.test_chain_ranges_gpu import tiled                                            # noqa: E402
from tests.test_instance_images_gpu import (BULK, CADENCE, FS, STALE, armed, drive, engine, is_q,   # noqa: E402
                                            params, run, same_out)

KINDS = ["f32f", "f32s", "q28"]
CASES = [("f32f", 1), ("f32f", 2), ("f32s", 1), ("f32s", 2), ("q28", 1)]   # (kind, DSPI_F32_CPL)
EINVAL, ERANGE = -22, -34


@pytest.fixture
def libm(oracle):
    oracle.set_libm_f64(1)
    yield oracle
    oracle.set_libm_f64(0)


def host_route(eng, src, dst):
    """What copy_instances replaces: one image per pair through host memory."""
    for s, d in zip(src, dst):
        eng.import_instances(eng.export_instances(int(s), 1), inst0=int(d))


def images(eng, chunk=512):
    """Whole-engine instance images, read in chunks (large engines)."""
    return np.concatenate([eng.export_instances(i, min(chunk, eng.n_instances - i)) for i in range(0, eng.n_instances, chunk)])


def digests(eng, chunk=512):
    """One digest per instance image (an 8192-instance float engine holds 1.3 GB of images)."""
    out = []
    for i in range(0, eng.n_instances, chunk):
        out += [hashlib.sha256(x.tobytes()).digest() for x in eng.export_instances(i, min(chunk, eng.n_instances - i))]
    return np.array(out, dtype=object)


def same_engine(a, b):
    return np.array_equal(images(a), images(b)) and np.array_equal(a.state_export(), b.state_export())


def _raw(eng, name, *args):
    return getattr(api.lib(), eng._PRE + "_" + name)(eng._h, *args)


def u32(xs):
    return (C.c_uint32 * max(len(xs), 1))(*[int(x) for x in xs])


def arm(eng, insts):
    st = np.zeros(1, L.PRESET_MUTE)
    st["smooth_gain"] = 1.0
    api.lib().dspi_preset_mute_arm(st.ctypes.data_as(C.c_void_p), int(FS))
    for i in insts:
        eng.set_preset_mute(st, FS, inst0=int(i))


# ---- 1. twin identity -------------------------------------------------------------------------------------------------------
# sources: stale (1), bulk-current (5, 8), unset (12, 33, 47); armed envelopes among sources (8, 12) and destinations (0, 40)
SRC = [1, 5, 8, 12, 33, 47]
DST = [40, 0, 63, 45, 9, 21]


@pytest.mark.parametrize("kind,cpl", CASES)
def test_copy_equals_the_host_image_route(libm, monkeypatch, kind, cpl):
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    a, b = engine(kind, 64), engine(kind, 64)
    try:
        chains = {12: None, 33: None}
        drive(libm, kind, a, 101, chains=chains)
        drive(libm, kind, b, 101)
        a.copy_instances(SRC, DST)
        host_route(b, SRC, DST)
        assert same_engine(a, b)
        ia = a.export_instances()
        assert np.array_equal(ia[DST], ia[SRC]), "a copy's image is its source's image"
        follow = {DST[SRC.index(s)]: chains[s] for s in chains}          # the oracle goes on from the copies
        for k in range(3):
            pcm = pcm_bytes(64, sum(CADENCE), 24, 110 + k)
            ra, rb = run(libm, kind, a, 0, follow, pcm), run(libm, kind, b, 0, None, pcm)
            assert same_out(ra, rb), f"call {k}"
        pcm = pcm_bytes(64, sum(CADENCE), 24, 119)
        sub_a, pdm_a, st_a = a.process_subframes_host(pcm, 24, CADENCE)
        sub_b, pdm_b, st_b = b.process_subframes_host(pcm, 24, CADENCE)
        assert np.array_equal(sub_a, sub_b) and np.array_equal(pdm_a, pdm_b) and st_a.tobytes() == st_b.tobytes()
        assert same_engine(a, b)
    finally:
        a.close()
        b.close()


# ---- 2. untouched instances -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_instances_outside_dst_are_untouched(libm, monkeypatch, kind, cpl):
    """Destinations mid-group (37, 38 share 32- and 64-row groups with non-destinations) and the last instance."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    a, u = engine(kind, 64), engine(kind, 64)
    src, dst = [3, 20, 6, 3], [37, 38, 63, 50]
    try:
        for e in (a, u):
            drive(libm, kind, e, 121)
        before = a.export_instances()
        a.copy_instances(src, dst)
        after = a.export_instances()
        keep = np.setdiff1d(np.arange(64), dst)
        assert np.array_equal(after[keep], before[keep])
        assert np.array_equal(after[dst], before[src])
        for k in range(2):
            pcm = pcm_bytes(64, sum(CADENCE), 24, 130 + k)
            pcm[dst] = pcm[src]
            ra, ru = run(libm, kind, a, 0, None, pcm), run(libm, kind, u, 0, None, pcm)
            assert same_out(ra, ru, keep, keep), f"call {k}: instances outside dst"
            assert same_out(ra, ru, dst, src), f"call {k}: copies against their sources in the untouched engine"
    finally:
        a.close()
        u.close()


# ---- 3. clone and scatter ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_clone_and_scattered_lists(oracle, kind):
    n = 2048
    a, b = engine(kind, n, 256), engine(kind, n, 256)
    rng = np.random.default_rng(141)
    try:
        P, bq = tiled(oracle, kind, n, FS, 141)
        for e in (a, b):
            e.set_params(P)
            e.upload_biquads(bq)
            arm(e, range(0, n, 7))
            e.process_packets_host(pcm_bytes(n, 192, 24, 142), 24, [96, 96])
        steps = [([7] * 17, rng.choice(np.arange(8, n), 17, replace=False))]                  # one source into 17 slots
        for m in (1, 17, 900):
            perm = rng.permutation(n)
            steps.append((rng.choice(perm[:m], m), perm[m:2 * m]))                              # sources repeat, scattered
        for src, dst in steps:
            a.copy_instances(src, dst)
            host_route(b, src, dst)
            assert same_engine(a, b), f"{len(src)} copies"
            pcm = pcm_bytes(n, 192, 24, 143 + len(src))
            assert same_out(a.process_packets_host(pcm, 24, [96, 96]), b.process_packets_host(pcm, 24, [96, 96]))
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("kind", KINDS)
def test_half_of_8192_instances_into_the_other_half(oracle, kind):
    n, h = 8192, 4096
    a = engine(kind, n, 192)
    rng = np.random.default_rng(151)
    try:
        P, bq = tiled(oracle, kind, n, FS, 151)
        a.set_params(P)
        a.upload_biquads(bq)
        a.process_packets_host(pcm_bytes(n, 192, 24, 152), 24, [96, 96])
        src, dst = rng.permutation(h), h + rng.permutation(h)
        ref = digests(a)
        a.copy_instances(src, dst)
        got = digests(a)
        assert (got[:h] == ref[:h]).all(), "sources changed"
        assert (got[dst] == ref[src]).all(), "copies differ from their sources"
        pcm = pcm_bytes(n, 192, 24, 153)
        pcm[dst] = pcm[src]
        sp, pd, st = a.process_packets_host(pcm, 24, [96, 96])
        assert np.array_equal(sp[dst], sp[src]) and np.array_equal(pd[dst], pd[src]) and st[dst].tobytes() == st[src].tobytes()
    finally:
        a.close()


# ---- 4. envelope accounting -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_envelope_mode_follows_the_copies(libm, kind):
    """One armed instance (5); copied over a plain one, then plain ones over both armed: the last envelope goes."""
    a, b = engine(kind, 64), engine(kind, 64)
    try:
        P, bq = params(libm, kind, 64, 161)
        for e in (a, b):
            e.set_params(P)
            e.upload_biquads(bq)
            arm(e, [5])
        for k, (src, dst) in enumerate([([5], [20]), ([30, 31], [5, 20])]):
            a.copy_instances(src, dst)
            host_route(b, src, dst)
            assert same_engine(a, b), f"step {k}"
            for j in range(3):                                               # the fade runs on across calls
                pcm = pcm_bytes(64, sum(CADENCE), 24, 170 + 10 * k + j)
                assert same_out(run(libm, kind, a, 0, None, pcm), run(libm, kind, b, 0, None, pcm)), f"step {k} call {j}"
                assert a.get_preset_mute().tobytes() == b.get_preset_mute().tobytes()
        arm(a, [40])                                                          # from none in envelope mode back to one
        arm(b, [40])
        a.copy_instances([40], [41])
        host_route(b, [40], [41])
        pcm = pcm_bytes(64, sum(CADENCE), 24, 199)
        assert same_out(run(libm, kind, a, 0, None, pcm), run(libm, kind, b, 0, None, pcm))
        assert a.get_preset_mute().tobytes() == b.get_preset_mute().tobytes()
    finally:
        a.close()
        b.close()


# ---- 5. EQ kernel choice ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_copies_that_make_and_break_one_band_topology(libm, monkeypatch, kind, cpl):
    """Every instance uniform but 61: copying a uniform instance over it gives the whole engine one band topology (the
    float EQ then runs its specialised kernel); spreading 61 instead breaks it in groups that had one.  The state blob
    holds the EQ topology words the kernel choice is made from."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    for src, dst in (([0], [61]), ([61, 61, 61], [5, 17, 40])):
        a, b = engine(kind, 64), engine(kind, 64)
        try:
            if is_q(kind):
                P, bq = params(libm, kind, 64, 181)
            else:
                from tests.chain_cases import chain_params
                P, bq = chain_params(libm, 64, FS, 181, uniform=True)
                Po, bqo = chain_params(libm, 64, FS, 182)
                P[61], bq[61] = Po[61], bqo[61]
            for e in (a, b):
                e.set_params(P)
                e.upload_biquads(bq)
                run(libm, kind, e, 183)
            a.copy_instances(src, dst)
            host_route(b, src, dst)
            assert same_engine(a, b), (src, dst)
            for k in range(2):
                pcm = pcm_bytes(64, sum(CADENCE), 24, 184 + k)
                assert same_out(run(libm, kind, a, 0, None, pcm), run(libm, kind, b, 0, None, pcm)), (src, dst, k)
        finally:
            a.close()
            b.close()


# ---- 6. ordering and follow-up calls ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_copy_is_ordered_behind_an_asynchronous_range_call(libm, kind):
    a, t = engine(kind, 64), engine(kind, 64)
    pairs = 2 if is_q(kind) else 4
    F = sum(CADENCE)
    src, dst = [2, 9, 30], [40, 33, 12]
    try:
        for e in (a, t):
            drive(libm, kind, e, 191)
        pcm = torch.from_numpy(pcm_bytes(32, F, 24, 192)).cuda()
        outs = {e: (torch.zeros((32, pairs, F, 2), dtype=torch.int32, device="cuda"), torch.zeros((32, F, 8), dtype=torch.int32, device="cuda"))
                for e in (a, t)}
        torch.cuda.synchronize()
        for e in (a, t):
            e.process_packets_range_device(0, 32, pcm.data_ptr(), 24, CADENCE, outs[e][0].data_ptr(), outs[e][1].data_ptr())
        a.copy_instances(src, dst)                                   # right behind the asynchronous call on [0, 32)
        t.sync()
        host_route(t, src, dst)
        assert same_engine(a, t)
        assert torch.equal(outs[a][0], outs[t][0]) and torch.equal(outs[a][1], outs[t][1])
    finally:
        a.close()
        t.close()


@pytest.mark.parametrize("kind", KINDS)
def test_record_and_mark_travel_with_the_copy(libm, kind):
    """collect_bulk_device and set_rate_device on copies of a current (6), a stale (2) and an unset (30) instance."""
    a, b = engine(kind, 64), engine(kind, 64)
    src, dst = [6, 2, 30], [50, 51, 52]
    try:
        for e in (a, b):
            drive(libm, kind, e, 201)
        assert 6 in BULK and 6 not in STALE and 2 in STALE and 30 not in BULK
        w0, h0, m0 = a.collect_bulk_device(0, 64)
        a.copy_instances(src, dst)
        host_route(b, src, dst)
        w1, h1, m1 = a.collect_bulk_device(0, 64)
        assert w1[dst].tobytes() == w0[src].tobytes() and h1[dst].tobytes() == h0[src].tobytes() and list(m1[dst]) == list(m0[src])
        assert list(m1[dst]) == [L.BULK_CURRENT, L.BULK_STALE, L.BULK_UNSET]
        rates = np.full(3, 44100.0, np.float32)
        ra, rb = a.set_rate_device(rates, inst0=50), b.set_rate_device(rates, inst0=50)
        assert list(ra) == list(rb) == list(m0[src])
        assert same_engine(a, b)
        pcm = pcm_bytes(64, sum(CADENCE), 24, 202)
        assert same_out(run(libm, kind, a, 0, None, pcm), run(libm, kind, b, 0, None, pcm))
    finally:
        a.close()
        b.close()


# ---- 7. refusals ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_refused_copies_change_nothing(oracle, kind):
    a = engine(kind, 40)
    try:
        P, bq = params(oracle, kind, 40, 211)
        a.set_params(P)
        a.upload_biquads(bq)
        arm(a, armed(40))
        a.process_packets_host(pcm_bytes(40, sum(CADENCE), 24, 212), 24, CADENCE)
        ref, blob = a.export_instances(), a.state_export()

        def refused(code, src, dst, n=None):
            n = len(src) if n is None else n
            s = src if src is None else u32(src)
            d = dst if dst is None else u32(dst)
            rc = _raw(a, "copy_instances", n, s, d)
            assert rc == code, (rc, api.lib().dspi_last_error())
            assert np.array_equal(a.export_instances(), ref) and np.array_equal(a.state_export(), blob)

        refused(EINVAL, None, [3], n=1)                                 # NULL lists
        refused(EINVAL, [3], None)
        refused(EINVAL, None, None, n=0)
        refused(ERANGE, [1, 40], [2, 3])                                # at n_instances
        refused(ERANGE, [1, 2], [3, 0xFFFFFFFF])
        refused(EINVAL, [1, 2, 4], [7, 8, 7])                           # a destination twice
        refused(EINVAL, [1, 2, 4], [7, 1, 9])                           # in both lists
        refused(EINVAL, [5], [5])
        refused(0, [1, 2], [3, 4], n=0)                                 # n == 0: nothing
        with pytest.raises(api.DspiError):
            a.copy_instances([1, 2], [3, 3])
        assert np.array_equal(a.export_instances(), ref)
    finally:
        a.close()
