"""GPU: per-instance lifecycle of the chain engines - dspi_chain(q)_export_instances / _import_instances / _reset_instances.
The source engine is driven through everything an instance carries first: bulk packets on some instances, set_params and
biquad uploads on others (current, stale and unset configuration records), preset-mute fades in progress, non-default
S/PDIF transmitters, output delays up to the ring size - 1, and calls on the 44.1 kHz packet cadence.  The bars are the
engine's own whole-engine calls (state blob, collect, transmitter, envelope, biquads), a twin engine, and the oracle."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                                  # noqa: E402
from tests.bulk_cases import wire_packet                                                 # noqa: E402
from tests.chain_cases import chain_params, chain_params_q28, pcm_bytes                  # noqa: E402
from tests.orc import arm_mute_envelope, make_orc_chain, make_orc_chain_q28             # noqa: E402

KINDS = ["f32f", "f32s", "q28"]
EINVAL, ERANGE = -22, -34
FS = 48000.0
CADENCE = [44] * 9 + [45]                      # 441 frames every 10 ms
BULK, STALE = range(0, 10), range(0, 4)        # bulk packets on [0, 10), then set_params again on [0, 4): stale; the rest unset


def is_q(kind):
    return kind == "q28"


def engine(kind, n, frames=1024, n_bands=L.NUM_BANDS):
    return api.ChainEngineQ28(n, max_frames=frames, n_bands=n_bands) if is_q(kind) else api.ChainEngine(kind, n, max_frames=frames)


def params(oracle, kind, n, seed, uniform=False):
    P, bq = chain_params_q28(oracle, n, FS, seed) if is_q(kind) else chain_params(oracle, n, FS, seed, uniform=uniform)
    n_out, mx = (5, L.CHAINQ_MAX_DELAY) if is_q(kind) else (9, L.CHAIN_MAX_DELAY)
    if not uniform:
        P["host_mute"] = 0
        for i in range(0, n, 3):                                   # delays up to the ring size - 1
            for o in range(n_out):
                P[i]["matrix"]["outputs"][o]["delay_samples"] = [mx - 1, 1, 0, mx // 2 + 7, 45][(o + i) % 5]
    return P, bq


def armed(n):
    return [i for i in range(n) if i % 4 == 0]


def drive(oracle, kind, eng, seed, calls=2, chains=None):
    """Configures `eng` (n >= 16) and runs `calls` calls on the 44.1 kHz cadence; returns the params, biquads and outputs.
    `chains` (dict instance -> oracle chain) are run along for instances outside BULK."""
    n = eng.n_instances
    P, bq = params(oracle, kind, n, seed)
    eng.set_params(P)
    eng.upload_biquads(bq)
    plat = L.PLATFORM_RP2040 if is_q(kind) else L.PLATFORM_RP2350
    w = np.concatenate([wire_packet(plat, seed * 100 + i) for i in BULK])
    assert (eng.apply_bulk_device(w, FS, inst0=BULK.start) == 0).all()
    eng.set_params(P[STALE.start:STALE.stop], inst0=STALE.start)
    eng.upload_biquads(bq[STALE.start:STALE.stop], inst0=STALE.start)
    st = np.zeros(1, L.PRESET_MUTE)
    st["smooth_gain"] = 1.0
    api.lib().dspi_preset_mute_arm(st.ctypes.data_as(C.c_void_p), int(FS))
    for i in armed(n):
        eng.set_preset_mute(st, FS, inst0=i)
    rng = np.random.default_rng(seed)
    eng.set_spdif_tx(rng.integers(0, 192, n), rng.integers(0, 256, (n, 5)).astype(np.uint8))
    chains = {} if chains is None else chains
    for i in list(chains):
        chains[i] = make_orc_chain_q28(oracle, P[i], bq[i]) if is_q(kind) else make_orc_chain(oracle, P[i], bq[i])
        if i in armed(n):
            arm_mute_envelope(chains[i], FS)
    outs = [run(oracle, kind, eng, seed + 1 + k, chains) for k in range(calls)]
    return P, bq, outs


def orc_packets(oracle, kind, chain, pcm, frames):
    F, bpf = int(sum(frames)), 6
    spdif = np.zeros((2 if is_q(kind) else 4, F, 2), np.int32)
    pdm = np.zeros((F, 8), np.uint32)
    fn = getattr(oracle.lib, "orc_q28_chain_packet" if is_q(kind) else f"orc_{kind}_chain_packet")
    data = np.ascontiguousarray(pcm)
    f0 = 0
    for k in frames:
        fn(C.addressof(chain), data.ctypes.data + f0 * bpf, int(k) * bpf, 24, spdif.ctypes.data + f0 * 8, F * 2, pdm.ctypes.data + f0 * 32)
        f0 += int(k)
    return spdif, pdm


def run(oracle, kind, eng, seed, chains=None, pcm=None):
    """One call on the cadence; the oracle chains (instance -> chain) run the same packets and must agree."""
    pcm = pcm_bytes(eng.n_instances, sum(CADENCE), 24, seed) if pcm is None else pcm
    spdif, pdm, status = eng.process_packets_host(pcm, 24, CADENCE)
    for i, ch in (chains or {}).items():
        ws, wp = orc_packets(oracle, kind, ch, pcm[i], CADENCE)
        assert np.array_equal(spdif[i], ws), f"instance {i}: S/PDIF words differ from the oracle"
        if int(ch.out[4 if is_q(kind) else 8].enabled):
            assert np.array_equal(pdm[i], wp), f"instance {i}: PDM differs from the oracle"
    return spdif, pdm, status


def same_out(a, b, sa=slice(None), sb=slice(None)):
    return all(np.array_equal(x[sa], y[sb]) for x, y in zip(a[:2], b[:2])) and a[2][sa].tobytes() == b[2][sb].tobytes()


def whole_engine(eng):
    w, hv, marks = eng.collect_bulk_device()
    return [eng.state_export(), w, hv, marks, eng.get_spdif_tx(), eng.get_preset_mute(), eng.download_biquads()]


@pytest.fixture
def libm(oracle):
    oracle.set_libm_f64(1)
    yield oracle
    oracle.set_libm_f64(0)


# ---- 1. full-engine identity: every field of every instance ---------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_all_instances_into_a_fresh_engine_give_the_same_engine(libm, kind):
    a, b = engine(kind, 64), engine(kind, 64)
    try:
        drive(libm, kind, a, 11)
        img = a.export_instances()
        assert img.shape == (64, a.instance_image_size())
        b.import_instances(img)
        for k, (x, y) in enumerate(zip(whole_engine(a), whole_engine(b))):
            assert x.tobytes() == y.tobytes(), f"whole-engine read {k} differs"
        marks = whole_engine(a)[3]
        assert set(marks[BULK.stop:]) == {L.BULK_UNSET} and set(marks[STALE.stop:BULK.stop]) == {L.BULK_CURRENT} and set(marks[STALE]) == {L.BULK_STALE}
        for k in range(2):
            pcm = pcm_bytes(64, sum(CADENCE), 24, 50 + k)
            assert same_out(a.process_packets_host(pcm, 24, CADENCE), b.process_packets_host(pcm, 24, CADENCE)), f"call {k}"
        assert np.array_equal(a.export_instances(), b.export_instances())
    finally:
        a.close()
        b.close()


# ---- 2. migration into an engine of another shape ----------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_moved_instances_continue_bit_exact(libm, kind):
    """[5, 14) of A -> [100, 109) of B (other n_instances and max_frames; B's own instances uniform, so its float EQ runs a
    specialised kernel).  Instance 12 (configured by set_params, an armed envelope) is also run by the oracle throughout."""
    a, b, twin = engine(kind, 64, 441), engine(kind, 160, 2048), engine(kind, 160, 2048)
    lo, hi, at, probe = 5, 14, 100, 12
    try:
        chains = {probe: None}
        drive(libm, kind, a, 21, chains=chains)
        Pb, bqb = chain_params_q28(libm, 160, FS, 22) if is_q(kind) else chain_params(libm, 160, FS, 22, uniform=True)
        for e in (b, twin):
            e.set_params(Pb)
            e.upload_biquads(bqb)
            run(libm, kind, e, 23)
        b.import_instances(a.export_instances(lo, hi - lo), inst0=at)
        assert np.array_equal(b.export_instances(at, hi - lo), a.export_instances(lo, hi - lo))
        done_a = done_b = None
        for k in range(4):
            pa = pcm_bytes(64, sum(CADENCE), 24, 60 + k)
            pb = pcm_bytes(160, sum(CADENCE), 24, 70 + k)
            pb[at:at + hi - lo] = pa[lo:hi]
            ra = run(libm, kind, a, 0, None, pa)
            rb = run(libm, kind, b, 0, {at + probe - lo: chains[probe]}, pb)     # the oracle goes on from the moved instance
            rt = run(libm, kind, twin, 0, None, pb)
            assert same_out(ra, rb, slice(lo, hi), slice(at, at + hi - lo)), f"call {k}: moved instances"
            others = np.r_[0:at, at + hi - lo:160]
            assert same_out(rb, rt, others, others), f"call {k}: B's own instances"
            ga, gb = a.get_preset_mute(hi - lo, lo), b.get_preset_mute(hi - lo, at)
            assert ga.tobytes() == gb.tobytes()
            if done_a is None and (ga["smooth_gain"][np.array(armed(64)[2:4]) - lo] == 1.0).all():
                done_a = k
            if done_b is None and (gb["smooth_gain"][np.array(armed(64)[2:4]) - lo] == 1.0).all():
                done_b = k
        assert done_a is not None and done_a == done_b, "the fade must finish, on the same call"
    finally:
        for e in (a, b, twin):
            e.close()


# ---- 3. round trip and neighbours --------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_round_trip_is_a_no_op_and_neighbours_are_untouched(libm, kind):
    a, twin, other = engine(kind, 64), engine(kind, 64), engine(kind, 64)
    try:
        for e in (a, twin):
            drive(libm, kind, e, 31)
        drive(libm, kind, other, 32)
        img = a.export_instances()
        a.import_instances(img)
        assert np.array_equal(a.export_instances(), img)
        pcm = pcm_bytes(64, sum(CADENCE), 24, 33)
        assert same_out(run(libm, kind, a, 0, None, pcm), run(libm, kind, twin, 0, None, pcm))
        # inside one 32-instance group (and one 64-channel K1 group of every EQ role)
        before = a.export_instances()
        x = other.export_instances(3, 5)
        a.import_instances(x, inst0=37)
        after = a.export_instances()
        keep = np.r_[0:37, 42:64]
        assert np.array_equal(after[keep], before[keep]) and np.array_equal(after[37:42], x)
        pcm = pcm_bytes(64, sum(CADENCE), 24, 34)
        ra, rt = run(libm, kind, a, 0, None, pcm), run(libm, kind, twin, 0, None, pcm)
        assert same_out(ra, rt, keep, keep)
    finally:
        for e in (a, twin, other):
            e.close()


# ---- 4. reset by range -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_reset_instances_is_reset_state_for_the_range(libm, kind):
    a, t, u = engine(kind, 64), engine(kind, 64), engine(kind, 64)
    i0, n = 7, 11
    try:
        for e in (a, t, u):
            drive(libm, kind, e, 41)
        before = a.export_instances()
        a.reset_instances(i0, n)
        t.reset_state()
        ia, it = a.export_instances(), t.export_instances()
        rng_, keep = slice(i0, i0 + n), np.r_[0:i0, i0 + n:64]
        assert np.array_equal(ia[rng_], it[rng_]) and np.array_equal(ia[keep], before[keep])
        assert not np.array_equal(ia[rng_], before[rng_])
        pcm = pcm_bytes(64, sum(CADENCE), 24, 42)
        ra, rt, ru = (run(libm, kind, e, 0, None, pcm) for e in (a, t, u))
        assert same_out(ra, rt, rng_, rng_) and same_out(ra, ru, keep, keep)
        ia = a.export_instances()
        a.reset_instances(5, 0)                                    # n == 0 does nothing
        assert np.array_equal(a.export_instances(), ia)
    finally:
        for e in (a, t, u):
            e.close()


# ---- 5. power-on slot ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_fresh_image_returns_a_slot_to_power_on(libm, kind):
    a, fresh = engine(kind, 64), engine(kind, 40, 512)
    try:
        drive(libm, kind, a, 51)
        blank = fresh.export_instances(0, 1)
        a.import_instances(blank, inst0=20)
        assert np.array_equal(a.export_instances(20, 1), blank)
        w, hv, marks = a.collect_bulk_device(20, 1)
        assert marks[0] == L.BULK_UNSET and not w.tobytes().strip(b"\0") and not hv.tobytes().strip(b"\0")
        assert a.get_spdif_tx(1, 20).tobytes() == fresh.get_spdif_tx(1, 0).tobytes()
        assert a.get_preset_mute(1, 20).tobytes() == fresh.get_preset_mute(1, 0).tobytes()
        assert a.download_biquads(1, 20).tobytes() == fresh.download_biquads(1, 0).tobytes()
        pa = pcm_bytes(64, sum(CADENCE), 24, 52)
        pf = pcm_bytes(40, sum(CADENCE), 24, 53)
        pf[0] = pa[20]
        assert same_out(run(libm, kind, a, 0, None, pa), run(libm, kind, fresh, 0, None, pf), slice(20, 21), slice(0, 1))
    finally:
        a.close()
        fresh.close()


# ---- 6. ordering behind asynchronous calls ------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_export_and_import_are_ordered_behind_asynchronous_calls(libm, kind):
    a, t, other = engine(kind, 64), engine(kind, 64), engine(kind, 64)
    pairs = 2 if is_q(kind) else 4
    F = sum(CADENCE)
    try:
        for e in (a, t):
            drive(libm, kind, e, 61)
        drive(libm, kind, other, 62)
        x = other.export_instances(0, 9)
        pcm = torch.from_numpy(pcm_bytes(64, F, 24, 63)).cuda()
        outs = {e: (torch.zeros((64, pairs, F, 2), dtype=torch.int32, device="cuda"), torch.zeros((64, F, 8), dtype=torch.int32, device="cuda"))
                for e in (a, t)}
        torch.cuda.synchronize()
        for e in (a, t):
            e.process_packets_device(pcm.data_ptr(), 24, CADENCE, outs[e][0].data_ptr(), outs[e][1].data_ptr())
        ea = a.export_instances()                                  # right behind the asynchronous call
        t.sync()
        assert np.array_equal(ea, t.export_instances())
        for e in (a, t):
            e.process_packets_device(pcm.data_ptr(), 24, CADENCE, outs[e][0].data_ptr(), outs[e][1].data_ptr())
        a.import_instances(x, inst0=30)                            # does not reach into the call issued before it
        a.sync()
        t.sync()
        assert torch.equal(outs[a][0], outs[t][0]) and torch.equal(outs[a][1], outs[t][1])
        assert np.array_equal(a.export_instances(30, 9), x)
    finally:
        for e in (a, t, other):
            e.close()


# ---- 7. many staging chunks --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_export_and_import_over_many_staging_chunks(oracle, kind):
    n = 3000 if is_q(kind) else 1000
    a, b = engine(kind, n, 256), engine(kind, n, 256)
    try:
        P, bq = params(oracle, kind, n, 71)
        a.set_params(P)
        a.upload_biquads(bq)
        a.process_packets_host(pcm_bytes(n, 192, 24, 72), 24, [96, 96])
        size = a.instance_image_size()
        chunk = (32 << 20) // size
        n_chunks = -(-n // chunk)
        assert n_chunks >= 4 and n % chunk, (size, chunk)
        l0 = a.launch_count
        img = a.export_instances()
        assert a.launch_count - l0 == n_chunks + 2                  # gather per chunk + one EQ unpack per sub-engine
        l0 = b.launch_count
        b.import_instances(img)
        assert b.launch_count - l0 >= n_chunks + 2
        assert np.array_equal(b.export_instances(), img)
    finally:
        a.close()
        b.close()


# ---- 8. rejections -----------------------------------------------------------------------------------------------------
def _raw(eng, name, *args):
    return getattr(api.lib(), eng._PRE + "_" + name)(eng._h, *args)


@pytest.mark.parametrize("kind", KINDS)
def test_bad_images_and_arguments_change_nothing(oracle, kind):
    a = engine(kind, 40)
    wrong = {"f32f": engine("q28", 8), "f32s": engine("f32f", 8), "q28": engine("f32f", 8)}[kind]
    try:
        P, bq = params(oracle, kind, 40, 81)
        a.set_params(P)
        a.upload_biquads(bq)
        a.process_packets_host(pcm_bytes(40, sum(CADENCE), 24, 82), 24, CADENCE)
        ref = a.export_instances()
        size = ref.shape[1]

        def rejected(code, images, inst0=0, n=None, stride=None):
            img = np.ascontiguousarray(images, np.uint8)
            n = img.shape[0] if n is None else n
            rc = _raw(a, "import_instances", inst0, n, img.ctypes.data_as(C.c_void_p), C.c_size_t(img.shape[1] if stride is None else stride))
            assert rc == code, (rc, api.lib().dspi_last_error())
            assert np.array_equal(a.export_instances(), ref)

        donor = ref[30:35].copy()                                       # accepted, these would change instances 5..9
        rejected(EINVAL, wrong.export_instances(0, 2), inst0=5)          # Q28 into float, fused into strict, float into Q28
        if kind == "f32s":                                              # same size, other rounding
            assert wrong.instance_image_size() == size
        for off, val in ((0, 0x12345678), (4, 2)):                      # magic, version
            bad = donor.copy()
            bad[:, off:off + 4] = np.frombuffer(np.uint32(val).tobytes(), np.uint8)
            rejected(EINVAL, bad, inst0=5)
        bad = donor.copy()
        bad[2, 0] ^= 1                                                  # one bad image in the middle of the call
        rejected(EINVAL, bad, inst0=5)
        rejected(EINVAL, donor, inst0=5, stride=size - 16)              # short stride
        rejected(ERANGE, donor, inst0=38)                               # past the end
        rejected(ERANGE, donor, inst0=0xFFFFFFF0, n=0x20)               # end wraps in 32 bits
        rejected(0, donor, inst0=5, n=0)                                # n == 0: nothing
        assert _raw(a, "import_instances", 0, 1, None, C.c_size_t(size)) == EINVAL
        buf = np.zeros((2, size), np.uint8)
        assert _raw(a, "export_instances", 0, 1, None, C.c_size_t(size)) == EINVAL
        assert _raw(a, "export_instances", 0, 1, buf.ctypes.data_as(C.c_void_p), C.c_size_t(size - 1)) == EINVAL
        assert _raw(a, "export_instances", 39, 2, buf.ctypes.data_as(C.c_void_p), C.c_size_t(size)) == ERANGE
        assert _raw(a, "export_instances", 0xFFFFFFFF, 2, buf.ctypes.data_as(C.c_void_p), C.c_size_t(size)) == ERANGE
        assert _raw(a, "export_instances", 3, 0, buf.ctypes.data_as(C.c_void_p), C.c_size_t(size)) == 0 and not buf.any()
        assert _raw(a, "reset_instances", 39, 2) == ERANGE and _raw(a, "reset_instances", 0xFFFFFFFF, 2) == ERANGE
        assert _raw(a, "reset_instances", 12, 0) == 0
        assert np.array_equal(a.export_instances(), ref)
        if is_q(kind):                                                  # another band count is another engine kind
            e8 = engine(kind, 8, n_bands=8)
            try:
                rejected(EINVAL, e8.export_instances(0, 1), inst0=3)
            finally:
                e8.close()
    finally:
        a.close()
        wrong.close()
