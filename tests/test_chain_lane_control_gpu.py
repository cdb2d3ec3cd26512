"""GPU: lane control calls, dspi_chain(q)_lane_edit_bulk_device / _lane_set_preset_mute / _lane_set_spdif_tx /
_lane_reset_instances - Console edits, preset-change fades, transmitter restamps and device restarts issued on a clock
group's lane, between its process calls, without a host synchronisation.  The bar is a twin engine that gets the same
calls in the same order, the process calls as range calls and the control calls as engine-level calls: every output
buffer, the biquads, the instance images, the state blob, the transmitters, the envelopes, the configuration records and
the edit marks must be byte-identical.  Float engines run in both K1 geometries."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                                  # noqa: E402
from tests.bulk_cases import wire_packet                                                 # noqa: E402
from tests.test_bulk_edit_gpu import random_edits                                        # noqa: E402
from tests.test_chain_lanes_gpu import BIG, CADENCE, PACED, Proc, configure, state       # noqa: E402
from tests.test_chain_ranges_gpu import CASES, KINDS, engine, params                    # noqa: E402

EINVAL, ERANGE = -22, -34
WINDOWS = [(0, 100, 44100.0, 11), (128, 64, 48000.0, 12), (192, 96, 96000.0, 13)]   # 44.1 kHz, paced 48 kHz, 96 x 96 frames
FREE = (100, 28)                                            # in no window; shares the 64-row K1 group [64, 128) with lane 0


def full_state(eng):
    return state(eng) + (eng.download_biquads().tobytes(),)


def apply_windows(eng, windows, seed):
    """current configuration records, so that edits take effect"""
    for i0, m, fs, s in windows:
        res = eng.apply_bulk_device(np.concatenate([wire_packet(eng._PLATFORM, seed + s * 1000 + i) for i in range(m)]), fs, inst0=i0)
        assert (res == 0).all()


def fade(fs, n, gain=1.0):
    st = np.zeros(n, L.PRESET_MUTE)
    for i in range(n):
        one = np.zeros(1, L.PRESET_MUTE)
        one["smooth_gain"] = gain
        api.lib().dspi_preset_mute_arm(one.ctypes.data_as(C.c_void_p), int(fs))
        st[i] = one[0]
    return st


class Ctl:
    """One control call on window k: issued on lane k of engine a, as an engine-level call on engine t."""

    def __init__(self, kind, k, what, args):
        self.k, self.what, self.args = k, what, args
        self.d_res = {w: torch.full((len(args[0]),), -99, dtype=torch.int32, device="cuda") for w in "at"} if what == "edit" else None
        self.host_res = None

    def issue(self, which, eng, lane_id=None):
        a = self.args
        if lane_id is None:
            if self.what == "edit":
                self.host_res = eng.edit_bulk_device(a[0], a[1])
            elif self.what == "fade":
                eng.set_preset_mute(a[0], a[1], inst0=a[2], n=a[3])
            elif self.what == "tx":
                eng.set_spdif_tx(a[0], a[1], inst0=a[2])
            else:
                eng.reset_instances(a[0], a[1])
            return
        if self.what == "edit":
            eng.lane_edit_bulk_device(lane_id, a[0], a[1], results_ptr=self.d_res[which].data_ptr())
        elif self.what == "fade":
            eng.lane_set_preset_mute(lane_id, a[0], a[1], a[2], a[3])
        elif self.what == "tx":
            eng.lane_set_spdif_tx(lane_id, a[0], a[1], a[2])
        else:
            eng.lane_reset_instances(lane_id, a[0], a[1])

    def same(self):
        return self.what != "edit" or np.array_equal(self.d_res["a"].cpu().numpy(), self.host_res)


def control_ops(kind, rng, k):
    """a Console edit burst, a fade arm or disarm, a transmitter restamp or a device restart inside window k"""
    i0, m, fs, _ = WINDOWS[k]
    c = int(rng.integers(5))
    if c <= 1:
        return Ctl(kind, k, "edit", (random_edits(rng, kind, list(range(i0, i0 + m)), int(rng.integers(1, 12))), fs))
    a = i0 + int(rng.integers(m))
    b = int(rng.integers(1, i0 + m - a + 1))
    if c == 2:
        return Ctl(kind, k, "fade", (fade(fs, b, float(rng.uniform(0.2, 1.0))) if rng.random() < 0.7 else None, fs, a, b))
    if c == 3:
        return Ctl(kind, k, "tx", (rng.integers(0, 192, b), rng.integers(0, 256, (b, 5)).astype(np.uint8), a))
    return Ctl(kind, k, "reset", (a, b))


def frames_of(k, r):
    return (CADENCE, PACED[r % 3], BIG[:24])[k]


# ---- 1. control calls on three lanes equal engine-level calls on a twin ---------------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_lane_control_calls_equal_engine_level_calls(oracle, monkeypatch, kind, cpl):
    """Three phases; in each, every lane gets process calls and control calls interleaved (edits of gains, crosspoints,
    mutes, host volume, crossfeed, EQ bands with topology flips and bypasses; fade arms and disarms; transmitter restamps;
    resets), issued across the lanes without a host synchronisation.  The twin gets the same calls in the same order.
    Between phases both engines are compared; instances outside every window must not change at all."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    n = 288
    a, t = engine(kind, n, sum(BIG)), engine(kind, n, sum(BIG))
    try:
        for e in (a, t):
            configure(e, oracle, kind, WINDOWS, armed=[3, 130, 200])
            apply_windows(e, WINDOWS, 5)
        free0 = a.export_instances(*FREE).tobytes()
        lanes = [a.lane_open(i0, m) for i0, m, _, _ in WINDOWS]
        rng = np.random.default_rng(40 + cpl)
        for phase in range(3):
            seq = []
            for r in range(3):
                for k in rng.permutation(3):
                    i0, m, _, _ = WINDOWS[k]
                    seq.append(Proc(kind, k, i0, m, frames_of(k, r), (24, 16)[(r + k) % 2], (r + k + phase) % 3 == 1, 1000 * phase + 10 * r + k))
                    for _ in range(int(rng.integers(1, 4))):
                        seq.append(control_ops(kind, rng, k))
            torch.cuda.synchronize()
            for x in seq:
                x.issue("a", a, lanes[x.lane if isinstance(x, Proc) else x.k])
            for x in seq:
                x.issue("t", t)
            for ln in lanes:
                a.lane_sync(ln)
            t.sync()
            for j, x in enumerate(seq):
                assert x.same(), f"phase {phase}, call {j} ({type(x).__name__} {getattr(x, 'what', '')}) differs from the twin"
            assert full_state(a) == full_state(t), f"phase {phase}"
            assert a.export_instances(*FREE).tobytes() == free0
    finally:
        a.close()
        t.close()


# ---- 2. a held lane does not hold the others ------------------------------------------------------------------------------
def _cuda_driver():
    try:
        return C.CDLL("libcuda.so.1")
    except OSError:
        pytest.skip("libcuda.so.1 not loadable")


@pytest.mark.parametrize("kind", KINDS)
def test_lane_control_calls_do_not_wait_for_other_lanes(oracle, kind):
    """Lane 0's stream is held by a host gate (a host function that waits for a flag, for at most 30 s, and then simply
    returns).  Lane 1's edit, fade arm and process call are issued and lane_sync(1) returns while the gate is still closed;
    then the gate opens and lane 0's outputs equal the twin's."""
    drv = _cuda_driver()
    n = 288
    a, t = engine(kind, n, sum(BIG)), engine(kind, n, sum(BIG))
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
        fs1 = WINDOWS[1][2]
        warm = Ctl(kind, 1, "edit", (L.bulk_edit(130, ("outputs", 0, "gain_db"), np.float32(-1.0)), fs1))
        held = Proc(kind, 0, 0, 100, CADENCE, 24, False, 81)
        edit = Ctl(kind, 1, "edit", (np.concatenate([L.bulk_edit(140, ("outputs", 2, "gain_db"), np.float32(-6.0)),
                                                     L.bulk_edit(141, ("eq", 0, 1), (L.PEAKING, (0, 0, 0), 900.0, 1.1, 5.0))]), fs1))
        arm = Ctl(kind, 1, "fade", (fade(fs1, 3), fs1, 150, 3))
        other = Proc(kind, 1, 128, 64, PACED[0], 24, False, 82)
        torch.cuda.synchronize()
        warm.issue("a", a, lanes[1])                                   # the lane's staging exists before the gate closes
        a.lane_sync(lanes[1])
        held.issue("a", a, lanes[0])
        assert drv.cuLaunchHostFunc(C.c_void_p(a.lane_stream(lanes[0])), hold, None) == 0
        assert entered.wait(30.0)
        t0 = time.monotonic()
        for x in (edit, arm, other):
            x.issue("a", a, lanes[1])
        a.lane_sync(lanes[1])
        assert not gate.is_set() and time.monotonic() - t0 < 25.0, "lane 1 waited for the held lane 0"
        gate.set()
        a.lane_sync(lanes[0])
        for x in (warm, held, edit, arm, other):
            x.issue("t", t)
        t.sync()
        assert held.same() and other.same() and edit.same() and warm.same()
        assert full_state(a) == full_state(t)
    finally:
        gate.set()
        a.close()
        t.close()


# ---- 3. a topology flip by a lane edit, followed by lane process calls only ----------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_lane_edit_topology_flip_keeps_the_kernel_choice(oracle, monkeypatch, kind, cpl):
    """Every instance starts from one configuration, so that a run-time specialised K1 is selected for its topology
    (DSPI_JIT=force).  A lane edit flips band topologies (SVF <-> TDF2, bypass) of part of the window and lane process calls
    follow with no engine-level call in between, so the lane keeps running the kernel selected before; the twin re-selects
    after its edit.  Outputs and state must be byte-identical."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    monkeypatch.setenv("DSPI_JIT", "force")
    n, fs = 256, 48000.0
    a, t = engine(kind, n, 512), engine(kind, n, 512)
    try:
        pk = np.repeat(wire_packet(a._PLATFORM, 77), n)
        for e in (a, t):
            P, bq = params(oracle, kind, n, fs, 21)
            e.set_params(P)
            assert (e.apply_bulk_device(pk, fs) == 0).all()
            e.process_packets_host(np.zeros((n, 96 * 4), np.uint8), 16, [96])        # the kernel choice is made here
        lanes = [a.lane_open(0, 128), a.lane_open(128, 128)]
        flips = np.concatenate([L.bulk_edit(i, ("eq", ch, b, "type"), [L.LOWPASS, L.PEAKING, L.FLAT][(i + b) % 3])
                                for i in range(0, 96, 3) for ch in (0, 1) for b in range(0, 10, 2)])
        seq = [Proc(kind, 0, 0, 128, [48] * 4, 24, False, 90), Ctl(kind, 0, "edit", (flips, fs))]
        seq += [Proc(kind, k, 128 * k, 128, [48] * 4, 24, r == 1, 91 + 2 * r + k) for r in range(3) for k in (0, 1)]
        torch.cuda.synchronize()
        for x in seq:
            x.issue("a", a, lanes[x.lane if isinstance(x, Proc) else x.k])
        for x in seq:
            x.issue("t", t)
        for ln in lanes:
            a.lane_sync(ln)
        t.sync()
        for j, x in enumerate(seq):
            assert x.same(), f"call {j}"
        assert full_state(a) == full_state(t)
    finally:
        a.close()
        t.close()


# ---- 4. refusals change nothing; launch counts after lanes -------------------------------------------------------------
def _raw(eng, name, *args):
    return getattr(api.lib(), eng._PRE + "_" + name)(*args)


@pytest.mark.parametrize("kind", KINDS)
def test_lane_control_refusals_change_nothing(oracle, kind):
    n, fs = 288, 48000.0
    a, t = engine(kind, n, 256), engine(kind, n, 256)
    try:
        for e in (a, t):
            configure(e, oracle, kind, [(0, n, fs, 31)], armed=[5, 70])
            apply_windows(e, [(0, n, fs, 31)], 8)
        h = a._h
        ok = a.lane_open(64, 100)                                     # window [64, 164)
        closed = a.lane_open(192, 64)
        a.lane_close(closed)
        res = torch.full((4,), 7, dtype=torch.int32, device="cuda")
        rp = C.c_void_p(res.data_ptr())
        good = L.bulk_edit(70, ("outputs", 0, "gain_db"), np.float32(-3.0))

        def edit(ln, e, rate=fs):
            e = np.ascontiguousarray(e)
            return _raw(a, "lane_edit_bulk_device", h, ln, int(e.size), e.ctypes.data_as(C.c_void_p), 0, C.c_float(rate), rp)

        outside = [L.bulk_edit(i, ("outputs", 0, "gain_db"), np.float32(-3.0)) for i in (63, 164, 200, 287)]
        bad_len = good.copy()
        bad_len["length"] = 25
        header = L.bulk_edit(70, ("outputs", 0, "gain_db"), np.float32(-3.0))
        header["offset"] = 4
        past = good.copy()
        past["instance"] = n
        assert edit(closed, good) == EINVAL and edit(16, good) == EINVAL
        assert _raw(a, "lane_edit_bulk_device", h, ok, 1, None, 0, C.c_float(fs), rp) == EINVAL
        assert edit(ok, good, rate=0.0) == EINVAL and edit(ok, good, rate=float("nan")) == EINVAL
        assert edit(ok, bad_len) == EINVAL and edit(ok, header) == EINVAL
        assert edit(ok, past) == ERANGE
        for o in outside:
            assert edit(ok, np.concatenate([good, o])) == ERANGE
        st = fade(fs, 4)
        sp = st.ctypes.data_as(C.c_void_p)
        tx = np.zeros(4, L.SPDIF_TX)
        tp = tx.ctypes.data_as(C.c_void_p)
        for ln, inst0, m, rc in ((closed, 64, 4, EINVAL), (16, 64, 4, EINVAL), (ok, 62, 4, ERANGE), (ok, 162, 4, ERANGE),
                                 (ok, 286, 4, ERANGE), (ok, 0xFFFFFFFE, 4, ERANGE)):
            assert _raw(a, "lane_set_preset_mute", h, ln, inst0, m, sp, int(fs)) == rc, (ln, inst0)
            assert _raw(a, "lane_set_preset_mute", h, ln, inst0, m, None, int(fs)) == rc, (ln, inst0)
            assert _raw(a, "lane_set_spdif_tx", h, ln, inst0, m, tp) == rc, (ln, inst0)
            assert _raw(a, "lane_reset_instances", h, ln, inst0, m) == rc, (ln, inst0)
        assert _raw(a, "lane_set_spdif_tx", h, ok, 64, 4, None) == EINVAL
        tx["block_pos"][2] = 192
        assert _raw(a, "lane_set_spdif_tx", h, ok, 64, 4, tp) == EINVAL
        l0 = a.launch_count
        for name in ("lane_set_preset_mute", "lane_set_spdif_tx", "lane_reset_instances"):
            args = {"lane_set_preset_mute": (sp, int(fs)), "lane_set_spdif_tx": (tp,), "lane_reset_instances": ()}[name]
            assert _raw(a, name, h, ok, 100, 0, *args) == 0               # n == 0 does nothing
        assert edit(ok, good[:0]) == 0
        assert a.launch_count == l0
        a.sync()
        assert res.tolist() == [7, 7, 7, 7]
        assert full_state(a) == full_state(t)
        # lanes used for control calls, then closed: every engine-level call issues what it issues on an engine that never had one
        ok2 = a.lane_open(192, 96)
        a.lane_edit_bulk_device(ok, np.concatenate([good, L.bulk_edit(80, ("eq", 0, 1, "type"), L.LOWPASS)]), fs)
        a.lane_set_preset_mute(ok2, fade(fs, 2), fs, 200)
        a.lane_set_spdif_tx(ok2, 9, bytes(5), 250)
        a.lane_reset_instances(ok, 100, 20)
        t.edit_bulk_device(np.concatenate([good, L.bulk_edit(80, ("eq", 0, 1, "type"), L.LOWPASS)]), fs)
        t.set_preset_mute(fade(fs, 2), fs, inst0=200)
        t.set_spdif_tx(9, bytes(5), inst0=250)
        t.reset_instances(100, 20)
        a.lane_close(ok)
        a.lane_close(ok2)
        calls = [lambda e: e.process_packets_host(np.zeros((n, 96 * 6), np.uint8), 24, [48, 48]),
                 lambda e: e.edit_bulk_device(L.bulk_edit(7, ("eq", 1, 2, "type"), L.HIGHPASS), fs),
                 lambda e: e.set_preset_mute(fade(fs, 3), fs, inst0=9),
                 lambda e: e.set_spdif_tx(3, bytes(5), inst0=11),
                 lambda e: e.reset_instances(0, 64),
                 lambda e: e.process_packets_host(np.zeros((n, 96 * 4), np.uint8), 16, [96])]
        for f in calls:
            counts = []
            for e in (t, a):
                c0 = e.launch_count
                f(e)
                counts.append(e.launch_count - c0)
            assert counts[0] == counts[1]
        assert full_state(a) == full_state(t)
    finally:
        a.close()
        t.close()
