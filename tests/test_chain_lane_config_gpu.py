"""GPU: lane configuration calls, dspi_chain(q)_lane_apply_bulk_device / _lane_apply_preset_device / _lane_set_rate_device -
a device connecting, a preset recall and a session rate change issued on a clock group's lane, between its process calls,
without a host synchronisation.  The bar is a twin engine that gets the same calls in the same order, the process calls
as range calls and the control calls as engine-level calls: every output buffer, the biquads, the instance images, the
state blob, the transmitters, the envelopes, the configuration records and every result code must be byte-identical.
Float engines run in both K1 geometries."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                                  # noqa: E402
from tests.bulk_cases import wire_packet                                                 # noqa: E402
from tests.test_chain_lane_control_gpu import (FREE, WINDOWS, Ctl, _cuda_driver, _raw, apply_windows, control_ops, fade,   # noqa: E402
                                               frames_of, full_state)
from tests.test_chain_lanes_gpu import BIG, CADENCE, PACED, Proc, configure              # noqa: E402
from tests.test_chain_ranges_gpu import CASES, KINDS, engine, params                    # noqa: E402
from tests.test_preset_device_gpu import fixture, padded, slot_size                      # noqa: E402

EINVAL, ERANGE = -22, -34
RATES = [44100.0, 48000.0, 96000.0]


def image_bank(kind, rng, count=24):
    """slot images: the reference's own, and images an engine collects from random packets, with their slot indices; then
    copies with a flipped CRC byte, a wrong magic, or a slot index other than the one they are loaded as (rejected)"""
    _, _, gold, gslots = fixture(kind)
    src = engine(kind, count, 64)
    try:
        assert not src.apply_bulk_device(np.concatenate([wire_packet(src._PLATFORM, 900 + i) for i in range(count)]), 48000.0).any()
        slots = rng.integers(0, 10, count).astype(np.uint8)
        imgs, marks = src.collect_preset_device(slots)
        assert (marks == L.BULK_CURRENT).all()
    finally:
        src.close()
    images, slots = np.concatenate([gold, imgs]), np.concatenate([gslots.astype(np.uint8), slots])
    bad = images[:6].copy()
    bad[0, 20] ^= 0x10                                          # CRC
    bad[1, 0] ^= 0x01                                           # magic
    bad_slots = slots[:6].copy()
    bad_slots[2] = (bad_slots[2] + 1) % 10                      # slot index
    bad[3, 9] ^= 0x80                                           # CRC word itself
    return np.concatenate([images, bad]), np.concatenate([slots, bad_slots])


class Cfg:
    """One configuration call on [i0, i0 + m) of window k: issued on lane k of engine a (device results), as an engine-level
    call on engine t (host results)."""

    def __init__(self, what, k, i0, args):
        self.what, self.k, self.i0, self.args = what, k, i0, args
        m = len(args[0])
        self.d_res = torch.full((m,), -99, dtype=torch.int32, device="cuda")
        self.host_res = None

    def issue(self, which, eng, lane_id=None):
        a = self.args
        if lane_id is None:
            if self.what == "apply":
                self.host_res = eng.apply_bulk_device(a[0], a[1], inst0=self.i0, host=a[2], exact_db=a[3])
            elif self.what == "preset":
                self.host_res = eng.apply_preset_device(a[0], a[1], inst0=self.i0, slots=a[2], master_volume_mode=a[3], host=a[4])
            else:
                self.host_res = eng.set_rate_device(a[0], inst0=self.i0)
            return
        ptr = self.d_res.data_ptr()
        if self.what == "apply":
            eng.lane_apply_bulk_device(lane_id, a[0], a[1], self.i0, host=a[2], exact_db=a[3], results_ptr=ptr)
        elif self.what == "preset":
            eng.lane_apply_preset_device(lane_id, a[0], a[1], self.i0, slots=a[2], master_volume_mode=a[3], host=a[4], results_ptr=ptr)
        else:
            eng.lane_set_rate_device(lane_id, a[0], self.i0, results_ptr=ptr)

    def same(self):
        return np.array_equal(self.d_res.cpu().numpy(), self.host_res)


def host_records(rng, m):
    hv = np.zeros(m, L.BULK_HOST)
    hv["volume_8_8"] = rng.integers(-32768, 32767, m)
    hv["host_mute"] = rng.random(m) < 0.2
    return hv


def config_op(kind, rng, k, bank, c=None):
    """a bulk apply of random packets (some rejected), a preset apply of bank images, or a rate switch, over part of window
    k; with `c` (0, 1, 2) that one over the whole window"""
    i0, m, fs, _ = WINDOWS[k]
    a = i0 if c is not None else i0 + int(rng.integers(m))
    b = m if c is not None else int(rng.integers(1, i0 + m - a + 1))
    c = int(rng.integers(3)) if c is None else c
    if c == 0:
        w = np.concatenate([wire_packet(L.PLATFORM_RP2040 if kind == "q28" else L.PLATFORM_RP2350, int(rng.integers(1 << 30))) for _ in range(b)])
        for j in np.flatnonzero(rng.random(b) < 0.25):       # rejected: -1 version, -2 platform, -3 channels, -4 length
            r = int(rng.integers(4))
            hd = w["header"]
            if r == 0:
                hd["format_version"][j] = 1
            elif r == 1:
                hd["platform_id"][j] ^= 1
            elif r == 2:
                hd["num_channels"][j] += 1
            else:
                hd["payload_length"][j] = 8
        return Cfg("apply", k, a, (w, fs, host_records(rng, b), bool(rng.integers(2))))
    if c == 1:
        images, slots = bank
        pick = rng.integers(0, images.shape[0], b)
        img = images[pick]
        if rng.integers(2):
            img = padded(img, 4096)
        return Cfg("preset", k, a, (img, fs, slots[pick], int(rng.integers(2)), host_records(rng, b)))
    return Cfg("rate", k, a, (rng.choice(RATES, b).astype(np.float32),))


def run_twins(a, t, seq, lanes):
    torch.cuda.synchronize()
    for x in seq:
        x.issue("a", a, lanes[x.lane if isinstance(x, Proc) else x.k])
    for x in seq:
        x.issue("t", t)
    for ln in set(lanes):
        a.lane_sync(ln)
    t.sync()
    for j, x in enumerate(seq):
        assert x.same(), f"call {j} ({type(x).__name__} {getattr(x, 'what', '')}) differs from the twin"
    assert full_state(a) == full_state(t)


def twins(kind, n=288, frames=sum(BIG)):
    return engine(kind, n, frames), engine(kind, n, frames)


# ---- 1. configuration calls on three lanes equal engine-level calls on a twin ---------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_lane_config_calls_equal_engine_level_calls(oracle, monkeypatch, kind, cpl):
    """Three phases; in each, every lane gets process calls, bulk applies, preset applies and rate switches interleaved
    with edits, fades, restamps and resets, issued across the lanes without a host synchronisation.  The 96 kHz group
    switches to 44.1 kHz and back (bands flip SVF <-> TDF2).  The twin gets the same calls in the same order."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    a, t = twins(kind)
    rng = np.random.default_rng(70 + cpl)
    bank = image_bank(kind, rng)
    try:
        for e in (a, t):
            configure(e, oracle, kind, WINDOWS, armed=[3, 130, 200])
            apply_windows(e, WINDOWS, 5)
        free0 = a.export_instances(*FREE).tobytes()
        lanes = [a.lane_open(i0, m) for i0, m, _, _ in WINDOWS]
        for phase in range(3):
            seq = []
            i2, m2 = WINDOWS[2][:2]
            seq.append(Cfg("rate", 2, i2, (np.full(m2, (44100.0, 96000.0, 44100.0)[phase], np.float32),)))
            for r in range(3):
                for k in rng.permutation(3):
                    i0, m, _, _ = WINDOWS[k]
                    seq.append(Proc(kind, k, i0, m, frames_of(k, r), (24, 16)[(r + k) % 2], (r + k + phase) % 3 == 1, 1000 * phase + 10 * r + k))
                    for _ in range(int(rng.integers(1, 4))):
                        seq.append(config_op(kind, rng, k, bank) if rng.random() < 0.6 else control_ops(kind, rng, k))
            run_twins(a, t, seq, lanes)
            assert a.export_instances(*FREE).tobytes() == free0, f"phase {phase}"
    finally:
        a.close()
        t.close()


# ---- 2. a preset change on one lane while another group runs -------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_preset_change_on_a_lane_while_another_group_runs(oracle, kind):
    """Lane 1: fade arm -> process -> lane preset apply -> disarm -> process, while lane 0 processes."""
    a, t = twins(kind)
    rng = np.random.default_rng(81)
    images, slots = image_bank(kind, rng)
    try:
        for e in (a, t):
            configure(e, oracle, kind, WINDOWS, armed=[])
            apply_windows(e, WINDOWS, 9)
        lanes = [a.lane_open(i0, m) for i0, m, _, _ in WINDOWS[:2]]
        i1, m1, fs1, _ = WINDOWS[1]
        pick = rng.integers(0, 28, m1)                              # good images only
        seq = [Proc(kind, 0, 0, 100, CADENCE, 24, False, 1),
               Ctl(kind, 1, "fade", (fade(fs1, m1, 1.0), fs1, i1, m1)),
               Proc(kind, 1, i1, m1, PACED[0], 24, False, 2),
               Proc(kind, 0, 0, 100, CADENCE, 24, True, 3),
               Cfg("preset", 1, i1, (images[pick], fs1, slots[pick], 1, host_records(rng, m1))),
               Ctl(kind, 1, "fade", (None, fs1, i1, m1)),
               Proc(kind, 0, 0, 100, CADENCE, 16, False, 4),
               Proc(kind, 1, i1, m1, PACED[1], 24, True, 5)]
        run_twins(a, t, seq, lanes)
        assert (seq[4].d_res.cpu().numpy() == 0).all()
    finally:
        a.close()
        t.close()


# ---- 3. a held lane does not hold the others ------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_lane_config_calls_do_not_wait_for_other_lanes(oracle, kind):
    """Lane 0's stream is held by a host gate (a host function that waits for a flag, for at most 30 s, and then simply
    returns).  Lane 1's bulk apply, preset apply, rate switch and process call are issued and lane_sync(1) returns while
    the gate is still closed; then the gate opens and both engines are compared."""
    drv = _cuda_driver()
    a, t = twins(kind)
    rng = np.random.default_rng(82)
    bank = image_bank(kind, rng)
    gate = threading.Event()
    entered = threading.Event()

    @C.CFUNCTYPE(None, C.c_void_p)
    def hold(_):
        entered.set()
        gate.wait(30.0)

    try:
        for e in (a, t):
            configure(e, oracle, kind, WINDOWS, armed=[3])
            apply_windows(e, WINDOWS, 6)
        lanes = [a.lane_open(i0, m) for i0, m, _, _ in WINDOWS[:2]]
        i1, m1, fs1, _ = WINDOWS[1]
        # the lane's staging exists, and every buffer of its ring has carried a whole-window apply (its largest upload),
        # before the gate closes
        warm = [config_op(kind, rng, 1, bank, c=1)] + [config_op(kind, rng, 1, bank, c=0) for _ in range(9)]
        for x in warm:
            x.issue("a", a, lanes[1])
        a.lane_sync(lanes[1])
        held = Proc(kind, 0, 0, 100, CADENCE, 24, False, 81)
        pick = rng.integers(0, bank[0].shape[0], m1)
        calls = [Cfg("apply", 1, i1 + 3, (np.concatenate([wire_packet(a._PLATFORM, 300 + i) for i in range(20)]), fs1, host_records(rng, 20), False)),
                 Cfg("preset", 1, i1, (bank[0][pick], fs1, bank[1][pick], 0, host_records(rng, m1))),
                 Cfg("rate", 1, i1 + 10, (np.full(30, 96000.0, np.float32),)),
                 Proc(kind, 1, i1, m1, PACED[0], 24, False, 82)]
        torch.cuda.synchronize()
        held.issue("a", a, lanes[0])
        assert drv.cuLaunchHostFunc(C.c_void_p(a.lane_stream(lanes[0])), hold, None) == 0
        assert entered.wait(30.0)
        t0 = time.monotonic()
        for x in calls:
            x.issue("a", a, lanes[1])
        a.lane_sync(lanes[1])
        assert not gate.is_set() and time.monotonic() - t0 < 25.0, "lane 1 waited for the held lane 0"
        gate.set()
        a.lane_sync(lanes[0])
        for x in warm + [held] + calls:
            x.issue("t", t)
        t.sync()
        for x in warm + [held] + calls:
            assert x.same()
        assert full_state(a) == full_state(t)
    finally:
        gate.set()
        a.close()
        t.close()


# ---- 4. calls across the staging chunk, many uploads in flight, caller buffers reused -------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_chunks_ring_and_reused_caller_buffers(oracle, kind):
    """A lane window of 1216 instances: a bulk apply over all of it and a preset apply over 1100 cross the 1024-instance
    staging chunk.  Then 14 small applies, preset applies and rate switches follow with no synchronisation, more than the
    ring's 8 buffers.  The caller's packets, host records, images and rates are overwritten as soon as each call returns."""
    n, fs = 1344, 48000.0
    a, t = engine(kind, n, 96), engine(kind, n, 96)
    rng = np.random.default_rng(83)
    images, slots = image_bank(kind, rng)
    try:
        for e in (a, t):
            P, bq = params(oracle, kind, n, fs, 17)
            e.set_params(P)
            e.upload_biquads(bq)
        lane = a.lane_open(64, 1216)
        plat = a._PLATFORM
        seq = [Cfg("apply", 0, 64, (np.concatenate([wire_packet(plat, 5000 + i) for i in range(1216)]), fs, host_records(rng, 1216), False))]
        pick = rng.integers(0, 28, 1100)
        seq.append(Cfg("preset", 0, 100, (padded(images[pick], 4096), fs, slots[pick], 1, host_records(rng, 1100))))
        for j in range(14):
            i0 = 64 + int(rng.integers(1100))
            m = int(rng.integers(1, 60))
            c = j % 3
            if c == 0:
                seq.append(Cfg("apply", 0, i0, (np.concatenate([wire_packet(plat, 7000 + 100 * j + i) for i in range(m)]), fs, host_records(rng, m), True)))
            elif c == 1:
                p = rng.integers(0, images.shape[0], m)
                seq.append(Cfg("preset", 0, i0, (images[p], fs, slots[p], 0, host_records(rng, m))))
            else:
                seq.append(Cfg("rate", 0, i0, (rng.choice(RATES, m).astype(np.float32),)))
        seq.append(Proc(kind, 0, 64, 1216, [48, 48], 24, True, 84))
        keep = [tuple(np.copy(v) if isinstance(v, np.ndarray) else v for v in x.args) if isinstance(x, Cfg) else None for x in seq]
        torch.cuda.synchronize()
        for x in seq:
            x.issue("a", a, lane)
            if isinstance(x, Cfg):
                for v in x.args:
                    if isinstance(v, np.ndarray):
                        v.view(np.uint8)[...] = 0x5A                    # the caller reuses its buffers at once
        for x, k in zip(seq, keep):
            if k is not None:
                x.args = k
            x.issue("t", t)
        a.lane_sync(lane)
        t.sync()
        for j, x in enumerate(seq):
            assert x.same(), f"call {j}"
        assert full_state(a) == full_state(t)
    finally:
        a.close()
        t.close()


# ---- 5. a topology flip by a lane rate switch, followed by lane process calls only ---------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_lane_rate_switch_keeps_the_kernel_choice(oracle, monkeypatch, kind, cpl):
    """Every instance starts from one 96 kHz configuration, so that a run-time specialised K1 is selected for its topology
    (DSPI_JIT=force).  A lane rate switch to 44.1 kHz flips the topology of bands between 5.9 and 12.8 kHz, and lane
    process calls follow with no engine-level call in between; the twin re-selects after its switch."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    monkeypatch.setenv("DSPI_JIT", "force")
    n, fs = 256, 96000.0
    a, t = engine(kind, n, 512), engine(kind, n, 512)
    try:
        pk = np.repeat(wire_packet(a._PLATFORM, 77), n)
        pk["eq"]["freq"][:, :, 1:10:2] = 9000.0
        for e in (a, t):
            P, bq = params(oracle, kind, n, fs, 21)
            e.set_params(P)
            assert (e.apply_bulk_device(pk, fs) == 0).all()
            e.process_packets_host(np.zeros((n, 96 * 4), np.uint8), 16, [96])        # the kernel choice is made here
        lanes = [a.lane_open(0, 128), a.lane_open(128, 128)]
        seq = [Proc(kind, 0, 0, 128, [48] * 4, 24, False, 90), Cfg("rate", 0, 0, (np.full(96, 44100.0, np.float32),))]
        seq += [Proc(kind, k, 128 * k, 128, [48] * 4, 24, r == 1, 91 + 2 * r + k) for r in range(3) for k in (0, 1)]
        run_twins(a, t, seq, lanes)
        assert (seq[1].d_res.cpu().numpy() == L.BULK_CURRENT).all()
    finally:
        a.close()
        t.close()


# ---- 6. refusals change nothing; launch counts with lanes open -----------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_lane_config_refusals_change_nothing(oracle, kind):
    n, fs = 288, 48000.0
    a, t = engine(kind, n, 256), engine(kind, n, 256)
    rng = np.random.default_rng(86)
    images, slots = image_bank(kind, rng)
    try:
        for e in (a, t):
            configure(e, oracle, kind, [(0, n, fs, 31)], armed=[5, 70])
            apply_windows(e, [(0, n, fs, 31)], 8)
        h = a._h
        ok = a.lane_open(64, 100)                                     # window [64, 164)
        closed = a.lane_open(192, 64)
        a.lane_close(closed)
        res = torch.full((8,), 7, dtype=torch.int32, device="cuda")
        rp = C.c_void_p(res.data_ptr())
        m = 4
        pk = np.concatenate([wire_packet(a._PLATFORM, 40 + i) for i in range(m)])
        hv = np.zeros(m, L.BULK_HOST)
        img = padded(images[:m], 4096)
        ld = np.zeros(m, L.PRESET_LOAD)
        ld["slot_index"] = slots[:m]
        rates = np.full(m, 44100.0, np.float32)
        P = lambda x: x.ctypes.data_as(C.c_void_p)                    # noqa: E731
        size = slot_size(kind)

        def apply(ln, inst0, cnt=m, p=P(pk), host=P(hv), rate=fs, out=rp):
            return _raw(a, "lane_apply_bulk_device", h, ln, inst0, cnt, p, host, 0, C.c_float(rate), out)

        def preset(ln, inst0, cnt=m, i=P(img), stride=4096, load=P(ld), host=P(hv), rate=fs, out=rp):
            return _raw(a, "lane_apply_preset_device", h, ln, inst0, cnt, i, C.c_size_t(stride), load, host, C.c_float(rate), out)

        def rate_sw(ln, inst0, cnt=m, r=P(rates), out=rp):
            return _raw(a, "lane_set_rate_device", h, ln, inst0, cnt, r, out)

        l0 = a.launch_count
        for ln, inst0, rc in ((closed, 64, EINVAL), (16, 64, EINVAL), (0xFFFFFFFF, 64, EINVAL), (ok, 62, ERANGE), (ok, 162, ERANGE),
                              (ok, 286, ERANGE), (ok, 0xFFFFFFFE, ERANGE)):
            assert apply(ln, inst0) == rc and preset(ln, inst0) == rc and rate_sw(ln, inst0) == rc, (ln, inst0)
        for kw in ({"p": None}, {"host": None}, {"out": None}, {"rate": 0.0}, {"rate": float("nan")}, {"rate": float("inf")}):
            assert apply(ok, 64, **kw) == EINVAL, kw
        for kw in ({"i": None}, {"load": None}, {"host": None}, {"out": None}, {"stride": size - 16}, {"rate": -1.0}):
            assert preset(ok, 64, **kw) == EINVAL, kw
        bad = np.full(40, 48000.0, np.float32)
        for v in (float("nan"), float("inf"), 0.0, -48000.0):
            bad[27] = v
            assert rate_sw(ok, 64, 40, P(bad)) == EINVAL, v
        assert rate_sw(ok, 64, r=None) == EINVAL
        assert apply(ok, 100, 0) == 0 and preset(ok, 100, 0) == 0 and rate_sw(ok, 100, 0) == 0 and rate_sw(ok, 100, 0, out=None) == 0
        assert a.launch_count == l0
        a.sync()
        assert res.tolist() == [7] * 8
        assert full_state(a) == full_state(t)
        # engine-level apply, preset apply and rate switch with lanes open issue what they issue on an engine without lanes
        ok2 = a.lane_open(192, 96)
        a.lane_apply_bulk_device(ok, pk, fs, 100, results_ptr=res.data_ptr())
        a.lane_set_rate_device(ok2, rates, 200)
        t.apply_bulk_device(pk, fs, inst0=100)
        t.set_rate_device(rates, inst0=200)
        a.sync()
        t.sync()
        calls = [lambda e: e.apply_bulk_device(pk, fs, inst0=10),
                 lambda e: e.apply_preset_device(img, fs, inst0=170, slots=slots[:m]),
                 lambda e: e.set_rate_device(rates, inst0=3),
                 lambda e: e.apply_preset_device(images[:40], fs, inst0=120, slots=slots[:40]),
                 lambda e: e.process_packets_host(np.zeros((n, 96 * 4), np.uint8), 16, [96])]
        for f in calls:
            counts = []
            for e in (t, a):
                c0 = e.launch_count
                f(e)
                counts.append(e.launch_count - c0)
            assert counts[0] == counts[1]
        a.lane_close(ok)
        a.lane_close(ok2)
        assert full_state(a) == full_state(t)
    finally:
        a.close()
        t.close()
