"""GPU: lane read calls, dspi_chain(q)_lane_collect_bulk_device / _lane_collect_preset_device / _lane_export_instances /
_lane_response_device / _lane_get_preset_mute / _lane_get_spdif_tx - a Console connecting, a preset save, an EQ curve, a
checkpoint and a fade or transmitter poll issued on a clock group's lane, between its process and control calls, without a
host synchronisation.  The bar is a twin engine that gets the same calls in the same order, the process calls as range
calls and the reads as engine-level getters: every read must give the twin's bytes, and leave the bytes around them (rows
past n, image stride tails, optional outputs not asked for) as they were.  A third engine gets the same sequence without
the reads: its outputs and state must equal the first's.  Float engines run in both K1 geometries.

The twin's collect, preset collect, export and response run the same kernels as the lane forms (bulk_collect_kernel,
preset_collect_kernel, instance_image_kernel, the response kernel), so for those reads these tests check ordering, staging,
addresses and the bytes left alone, not the content itself, which their own suites check against the oracle and the
reference.  The preset-mute and transmitter records come from new kernels and are checked against the host packing."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import layouts as L                                                       # noqa: E402
from tests.test_chain_lane_config_gpu import config_op, image_bank, twins               # noqa: E402
from tests.test_chain_lane_control_gpu import (WINDOWS, Ctl, _cuda_driver, _raw, apply_windows, control_ops, frames_of,   # noqa: E402
                                               full_state)
from tests.test_chain_lanes_gpu import BIG, CADENCE, PACED, Proc, configure              # noqa: E402
from tests.test_chain_ranges_gpu import CASES, KINDS, engine                             # noqa: E402
from tests.test_preset_device_gpu import slot_size                                        # noqa: E402

EINVAL, ERANGE = -22, -34
SENT = 0x5A
READS = ["bulk", "preset", "export", "resp", "mute", "tx"]


class Rd:
    """One read of [i0, i0 + m): issued on a lane of engine a into device buffers prefilled with SENT (two rows past m; a
    stride tail on the images), and as the engine-level getter on engine t (host memory)."""

    def __init__(self, eng, kind, what, k, i0, m, rng, fs=48000.0):
        self.what, self.k, self.i0, self.m, self.fs = what, k, i0, m, fs
        self.slots = rng.integers(0, 10, m).astype(np.uint8)
        self.freqs = np.sort(rng.uniform(0.0, fs / 2, int(rng.integers(1, 300)))).astype(np.float32)
        self.freqs[0] = 0.0
        want = [bool(x) for x in rng.random(2) < 0.7]      # the optional outputs asked for
        pad = 16 * int(rng.integers(0, 3))
        rows = {"bulk": [L.WIRE_BULK.itemsize] + [L.BULK_HOST.itemsize] * want[0] + [4] * want[1],
                "preset": [slot_size(kind)] + [4] * want[1],
                "export": [eng.instance_image_size()],
                "resp": [eng._OUTS * 2 * self.freqs.size * 8],
                "mute": [L.PRESET_MUTE.itemsize],
                "tx": [L.SPDIF_TX.itemsize]}[what]
        self.want = want
        self.row = rows                                     # bytes of each output per instance
        self.stride = [r + (pad if j == 0 and what in ("preset", "export") else 0) for j, r in enumerate(rows)]
        self.buf = [torch.full(((m + 2) * s,), SENT, dtype=torch.uint8, device="cuda") for s in self.stride]
        self.host = None

    def ptrs(self):
        return [b.data_ptr() for b in self.buf]

    def issue(self, which, eng, lane_id=None):
        i0, m = self.i0, self.m
        if lane_id is None:
            if self.what == "bulk":
                w, h, r = eng.collect_bulk_device(i0, m)
                self.host = [w, h if self.want[0] else None, r if self.want[1] else None]
            elif self.what == "preset":
                img, r = eng.collect_preset_device(self.slots, i0, m)
                self.host = [img, r if self.want[1] else None]
            elif self.what == "export":
                self.host = [eng.export_instances(i0, m)]
            elif self.what == "resp":
                self.host = [eng.response(self.freqs, self.fs, i0, m)]
            elif self.what == "mute":
                self.host = [eng.get_preset_mute(m, i0)]
            else:
                self.host = [eng.get_spdif_tx(m, i0)]
            return
        p = self.ptrs()
        slots, freqs = self.slots.copy(), self.freqs.copy()
        if self.what == "bulk":
            it = iter(p[1:])
            h = next(it) if self.want[0] else 0
            r = next(it) if self.want[1] else 0
            eng.lane_collect_bulk_device(lane_id, i0, m, p[0], h, r)
        elif self.what == "preset":
            eng.lane_collect_preset_device(lane_id, slots, i0, p[0], self.stride[0], n=m, results_ptr=p[1] if self.want[1] else 0)
        elif self.what == "export":
            eng.lane_export_instances(lane_id, i0, m, p[0], self.stride[0])
        elif self.what == "resp":
            eng.lane_response_device(lane_id, freqs, self.fs, i0, m, p[0])
        elif self.what == "mute":
            eng.lane_get_preset_mute(lane_id, i0, m, p[0])
        else:
            eng.lane_get_spdif_tx(lane_id, i0, m, p[0])
        slots[...] = 0xEE                                   # the caller reuses its host inputs at once
        freqs[...] = np.nan

    def expected(self):
        out = []
        got = [h for h in self.host if h is not None]
        for h, row, s in zip(got, self.row, self.stride):
            e = np.full((self.m + 2, s), SENT, np.uint8)
            e[:self.m, :row] = np.frombuffer(np.ascontiguousarray(h).tobytes(), np.uint8).reshape(self.m, row)
            out.append(e.reshape(-1))
        return out

    def same(self):
        return all(np.array_equal(b.cpu().numpy(), e) for b, e in zip(self.buf, self.expected()))


def read_op(eng, kind, rng, k, what=None):
    i0, m, fs, _ = WINDOWS[k]
    a = i0 + int(rng.integers(m))
    b = int(rng.integers(1, i0 + m - a + 1))
    return Rd(eng, kind, what or READS[int(rng.integers(len(READS)))], k, a, b, rng, fs)


def run_seq(eng, seq, lanes, which):
    for x in seq:
        x.issue(which, eng, lanes[x.lane if isinstance(x, Proc) else x.k])
    for ln in set(lanes):
        eng.lane_sync(ln)


def for_r(seq):
    """outputs of a third engine for the process calls and lane edits of seq"""
    for x in seq:
        if isinstance(x, Proc):
            x.out["r"] = tuple(torch.zeros_like(v) if v is not None else None for v in x.out["a"])
        elif isinstance(x, Ctl) and x.d_res is not None:
            x.d_res["r"] = torch.full_like(x.d_res["a"], -99)


# ---- 1. reads on three lanes equal engine-level reads on a twin, and change nothing ----------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_lane_reads_equal_engine_level_reads(oracle, monkeypatch, kind, cpl):
    """Two phases; in each, every lane gets process calls (mixed cadences), control and configuration calls and every kind
    of read, interleaved across the lanes without a host synchronisation.  Engine t gets the same calls in the same order
    with the reads as engine-level getters; engine r gets the same sequence on its lanes without any read."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    a, t = twins(kind)
    r = engine(kind, a.n_instances, sum(BIG))
    rng = np.random.default_rng(90 + cpl)
    bank = image_bank(kind, rng)
    try:
        for e in (a, t, r):
            configure(e, oracle, kind, WINDOWS, armed=[3, 130, 200])
            apply_windows(e, WINDOWS, 5)
        lanes = [a.lane_open(i0, m) for i0, m, _, _ in WINDOWS]
        rlanes = [r.lane_open(i0, m) for i0, m, _, _ in WINDOWS]
        for phase in range(2):
            seq = []
            for rr in range(3):
                for k in rng.permutation(3):
                    i0, m, _, _ = WINDOWS[k]
                    seq.append(Proc(kind, k, i0, m, frames_of(k, rr), (24, 16)[(rr + k) % 2], (rr + k + phase) % 3 == 1, 2000 * phase + 10 * rr + k))
                    for _ in range(int(rng.integers(2, 5))):
                        u = rng.random()
                        seq.append(read_op(a, kind, rng, k) if u < 0.45 else config_op(kind, rng, k, bank) if u < 0.7 else control_ops(kind, rng, k))
            for what in READS:                                              # every kind at least once per phase
                seq.insert(int(rng.integers(len(seq) + 1)), read_op(a, kind, rng, int(rng.integers(3)), what))
            writes = [x for x in seq if not isinstance(x, Rd)]
            for_r(writes)
            torch.cuda.synchronize()
            run_seq(a, seq, lanes, "a")
            for x in seq:
                x.issue("t", t)
            t.sync()
            for j, x in enumerate(seq):
                assert x.same(), f"phase {phase}, call {j} ({type(x).__name__} {getattr(x, 'what', '')}) differs from the twin"
            assert full_state(a) == full_state(t), f"phase {phase}"
            run_seq(r, writes, rlanes, "r")
            for x in writes:
                if isinstance(x, Proc):
                    assert all((u is None and v is None) or torch.equal(u, v) for u, v in zip(x.out["a"], x.out["r"])), "a read changed a process call"
            assert full_state(r) == full_state(a), f"phase {phase}: a read changed the engine"
    finally:
        for e in (a, t, r):
            e.close()


# ---- 2. a held lane does not hold the reads of another ---------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_lane_reads_do_not_wait_for_other_lanes(oracle, kind):
    """Lane 0's stream is held by a host gate (a host function that waits for a flag, for at most 30 s, and then simply
    returns).  Every read is issued on lane 1 and lane_sync(1) returns while the gate is still closed; then the gate opens
    and the results equal the twin's."""
    drv = _cuda_driver()
    a, t = twins(kind)
    rng = np.random.default_rng(92)
    gate = threading.Event()
    entered = threading.Event()

    @C.CFUNCTYPE(None, C.c_void_p)
    def hold(_):
        entered.set()
        gate.wait(30.0)

    try:
        for e in (a, t):
            configure(e, oracle, kind, WINDOWS, armed=[3, 130])
            apply_windows(e, WINDOWS, 6)
        lanes = [a.lane_open(i0, m) for i0, m, _, _ in WINDOWS[:2]]
        warm = [read_op(a, kind, rng, 1, w) for w in ("preset", "export", "resp")]   # the lane's staging and table exist
        for x in warm:
            x.issue("a", a, lanes[1])
        a.lane_sync(lanes[1])
        held = Proc(kind, 0, 0, 100, CADENCE, 24, False, 91)
        calls = [read_op(a, kind, rng, 1, w) for w in READS] + [Proc(kind, 1, 128, 64, PACED[0], 24, False, 92)]
        calls += [read_op(a, kind, rng, 1, w) for w in READS]
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
        for j, x in enumerate(warm + [held] + calls):
            assert x.same(), j
        assert full_state(a) == full_state(t)
    finally:
        gate.set()
        a.close()
        t.close()


# ---- 3. a device moves to another engine without stopping its group --------------------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_lane_export_moves_a_group_to_another_engine(oracle, monkeypatch, kind, cpl):
    """Lane 1's window [128, 192) of engine A is exported on the lane, between its process calls, copied to the host and
    imported at [64, 128) of engine B.  B's next process calls give the bytes A's give."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    A = engine(kind, 288, sum(BIG))
    B = engine(kind, 128, sum(BIG))
    try:
        configure(A, oracle, kind, WINDOWS, armed=[3, 130, 150])
        apply_windows(A, WINDOWS, 7)
        lanes = [A.lane_open(i0, m) for i0, m, _, _ in WINDOWS]
        size = A.instance_image_size()
        imgs = torch.full((64 * (size + 32),), SENT, dtype=torch.uint8, device="cuda")
        seq = [Proc(kind, 1, 128, 64, PACED[0], 24, False, 93), Proc(kind, 0, 0, 100, CADENCE, 16, True, 94)]
        nxt = [Proc(kind, 1, 128, 64, PACED[r % 3], (24, 16)[r % 2], r == 1, 95 + r) for r in range(3)]
        torch.cuda.synchronize()
        for x in seq:
            x.issue("a", A, lanes[x.lane])
        A.lane_export_instances(lanes[1], 128, 64, imgs.data_ptr(), size + 32)
        for x in nxt:
            x.issue("a", A, lanes[1])
        A.lane_sync(lanes[1])
        host = imgs.cpu().numpy().reshape(64, size + 32)
        assert (host[:, size:] == SENT).all()
        B.import_instances(host, inst0=64)
        for x in nxt:
            x.inst0 = 64
            x.issue("t", B)
        B.sync()
        for j, x in enumerate(nxt):
            assert x.same(), f"process call {j} after the move"
    finally:
        A.close()
        B.close()


# ---- 4. refusals write nothing and leave the lane working ------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_lane_read_refusals_change_nothing(oracle, kind):
    n, fs = 288, 48000.0
    a, t = engine(kind, n, 256), engine(kind, n, 256)
    rng = np.random.default_rng(96)
    try:
        for e in (a, t):
            configure(e, oracle, kind, [(0, n, fs, 31)], armed=[5, 70])
            apply_windows(e, [(0, n, fs, 31)], 8)
        h = a._h
        ok = a.lane_open(64, 100)                                     # window [64, 164)
        closed = a.lane_open(192, 64)
        a.lane_close(closed)
        size, slot = a.instance_image_size(), slot_size(kind)
        out = torch.full((4 * size,), SENT, dtype=torch.uint8, device="cuda")
        o = C.c_void_p(out.data_ptr())
        slots = np.zeros(4, np.uint8)
        freqs = np.array([0.0, 1000.0, 24000.0], np.float32)
        S, F = slots.ctypes.data_as(C.c_void_p), freqs.ctypes.data_as(C.c_void_p)

        def calls(ln, inst0, cnt=2, p=o, hp=o, rp=o, s=S, stride=None, f=F, nf=3, rate=fs, only=range(6)):
            """the six reads with these arguments, or those of `only`"""
            fns = [lambda: _raw(a, "lane_collect_bulk_device", h, ln, inst0, cnt, p, hp, rp),
                   lambda: _raw(a, "lane_collect_preset_device", h, ln, inst0, cnt, s, p, C.c_size_t(stride or slot), rp),
                   lambda: _raw(a, "lane_export_instances", h, ln, inst0, cnt, p, C.c_size_t(stride or size)),
                   lambda: _raw(a, "lane_response_device", h, ln, inst0, cnt, f, nf, C.c_float(rate), p),
                   lambda: _raw(a, "lane_get_preset_mute", h, ln, inst0, cnt, p),
                   lambda: _raw(a, "lane_get_spdif_tx", h, ln, inst0, cnt, p)]
            return [fns[j]() for j in only]

        l0 = a.launch_count
        for ln, inst0, rc in ((closed, 64, EINVAL), (16, 64, EINVAL), (0xFFFFFFFF, 64, EINVAL), (ok, 62, ERANGE), (ok, 163, ERANGE),
                              (ok, 286, ERANGE), (ok, 0xFFFFFFFF, ERANGE)):
            assert calls(ln, inst0) == [rc] * 6, (ln, inst0)
        assert calls(ok, 64, p=None) == [EINVAL] * 6
        assert calls(ok, 64, s=None, only=[1]) == [EINVAL]
        assert calls(ok, 64, stride=slot - 16, only=[1]) == [EINVAL]
        assert calls(ok, 64, stride=size - 16, only=[2]) == [EINVAL]
        bad = freqs.copy()
        for f, nf, rate in ((None, 3, fs), (F, 0, fs), (F, 3, 0.0), (F, 3, float("nan")), (F, 3, 40000.0)):
            assert calls(ok, 64, f=f, nf=nf, rate=rate, only=[3]) == [EINVAL], (nf, rate)
        for v in (float("nan"), -1.0, 24000.5):
            bad[1] = v
            assert calls(ok, 64, f=bad.ctypes.data_as(C.c_void_p), only=[3]) == [EINVAL], v
        assert calls(ok, 100, cnt=0) == [0] * 6
        assert a.launch_count == l0
        a.sync()
        assert (out.cpu().numpy() == SENT).all()
        # the lane still works, and its reads equal the engine-level ones
        after = [Rd(a, kind, w, 0, 70 + 3 * j, 5, rng, fs) for j, w in enumerate(READS)]
        torch.cuda.synchronize()
        for x in after:
            x.issue("a", a, ok)
            x.issue("t", t)
        a.lane_sync(ok)
        for x in after:
            assert x.same(), x.what
        assert full_state(a) == full_state(t)
    finally:
        a.close()
        t.close()


# ---- 5. packets at any address; a response array that is not 8-byte aligned ----------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_lane_collect_at_any_packet_address(oracle, kind):
    """dspi_wire_bulk_params is packed, so a caller's packets may start at any byte (a reply buffer with a wire header in
    front of the payload).  Lane collects into packets at offsets 1, 4, 8 and 20 from an aligned base - the first one on a
    lane whose staging does not exist yet - between process calls, equal the twin's collects, and the bytes around them
    are left alone.  A lane response into an array that is not 8-byte aligned is refused and writes nothing."""
    n, fs = 288, 48000.0
    a, t = engine(kind, n, 256), engine(kind, n, 256)
    try:
        for e in (a, t):
            configure(e, oracle, kind, [(0, n, fs, 41)], armed=[70])
            apply_windows(e, [(0, n, fs, 41)], 3)
        lane = a.lane_open(64, 100)
        P = L.WIRE_BULK.itemsize
        cases = [(1, 66, 5), (4, 100, 37), (8, 64, 100), (20, 163, 1)]
        bufs = [(torch.full((off + (m + 2) * P,), SENT, dtype=torch.uint8, device="cuda"),
                 torch.full((m + 2, L.BULK_HOST.itemsize), SENT, dtype=torch.uint8, device="cuda"),
                 torch.full((m + 2,), -7, dtype=torch.int32, device="cuda")) for off, _, m in cases]
        procs = [Proc(kind, 0, 64, 100, [48, 48], 24, False, 300 + j) for j in range(len(cases))]
        torch.cuda.synchronize()
        for (off, i0, m), (pk, hv, res), pr in zip(cases, bufs, procs):
            pr.issue("a", a, lane)
            a.lane_collect_bulk_device(lane, i0, m, pk.data_ptr() + off, hv.data_ptr(), res.data_ptr())
        a.lane_sync(lane)
        for (off, i0, m), (pk, hv, res), pr in zip(cases, bufs, procs):
            pr.issue("t", t)
            w, h, r = t.collect_bulk_device(i0, m)
            got = pk.cpu().numpy()
            assert (got[:off] == SENT).all() and (got[off + m * P:] == SENT).all(), off
            assert got[off:off + m * P].tobytes() == w.tobytes(), off
            assert hv.cpu().numpy()[:m].tobytes() == h.tobytes() and (hv.cpu().numpy()[m:] == SENT).all(), off
            assert np.array_equal(res.cpu().numpy()[:m], r) and (res.cpu().numpy()[m:] == -7).all(), off
        t.sync()
        for pr in procs:
            assert pr.same()
        out = torch.full((4 * a._OUTS * 2 * 3 * 8 + 16,), SENT, dtype=torch.uint8, device="cuda")
        freqs = np.array([0.0, 1000.0, 24000.0], np.float32)
        l0 = a.launch_count
        for off in (4, 12):
            assert _raw(a, "lane_response_device", a._h, lane, 64, 2, freqs.ctypes.data_as(C.c_void_p), 3, C.c_float(fs),
                        C.c_void_p(out.data_ptr() + off)) == EINVAL
        assert a.launch_count == l0
        a.lane_response_device(lane, freqs, fs, 64, 2, out.data_ptr() + 8)
        a.lane_sync(lane)
        got = out.cpu().numpy()
        assert (got[:8] == SENT).all()
        assert got[8:8 + 2 * a._OUTS * 2 * 3 * 8].tobytes() == t.response(freqs, fs, 64, 2).tobytes()
        assert full_state(a) == full_state(t)
    finally:
        a.close()
        t.close()
