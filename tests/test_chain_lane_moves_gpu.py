"""GPU: lane move calls, dspi_chain(q)_lane_import_instances / _lane_copy_instances - a device moving into a clock group's
window (a rate change into another group, a move from another engine, a checkpoint restored into a running group) issued on
the groups' lanes, between their process, control, configuration and read calls, without a host synchronisation.  The bar
is a twin engine that gets the same calls in the same order, the process calls as range calls and every other call as an
engine-level call: every output buffer, the biquads, the instance images, the state blob, the transmitters, the envelopes,
the configuration records and every result are byte-identical.  Float engines run in both K1 geometries."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from tests.test_chain_lane_config_gpu import Cfg, config_op, image_bank, twins          # noqa: E402
from tests.test_chain_lane_control_gpu import (FREE, WINDOWS, Ctl, _cuda_driver, _raw, apply_windows, control_ops, fade,   # noqa: E402
                                               frames_of, full_state)
from tests.test_chain_lane_read_gpu import SENT, read_op                                  # noqa: E402
from tests.test_chain_lanes_gpu import BIG, CADENCE, PACED, Proc, configure              # noqa: E402
from tests.test_chain_ranges_gpu import CASES, KINDS, engine                             # noqa: E402
from tests.test_preset_device_gpu import padded                                           # noqa: E402

EINVAL, ERANGE = -22, -34
NOT_READY = 600                                             # CUDA_ERROR_NOT_READY


class Mv:
    """One move: an import of `images` at inst0 on lane kd, or a copy of src -> dst from lane ks to lane kd; on the twin the
    engine-level call.  With `raw` the lane call goes straight to the entry point with the test's own buffers, which are
    overwritten as soon as it returns."""

    def __init__(self, what, ks, kd, args, raw=False):
        self.what, self.ks, self.kd, self.raw = what, ks, kd, raw
        if what == "import":
            self.args = (np.ascontiguousarray(args[0], np.uint8), int(args[1]))
        else:
            self.args = tuple(np.ascontiguousarray(np.asarray(v).reshape(-1), np.uint32) for v in args)

    def issue(self, eng, lanes=None):
        a = self.args
        if lanes is None:
            if self.what == "import":
                eng.import_instances(a[0], inst0=a[1])
            else:
                eng.copy_instances(a[0], a[1])
            return
        if not self.raw:
            if self.what == "import":
                eng.lane_import_instances(lanes[self.kd], a[0], a[1])
            else:
                eng.lane_copy_instances(lanes[self.ks], lanes[self.kd], a[0], a[1])
            return
        buf = [np.copy(v) if isinstance(v, np.ndarray) else v for v in a]
        P = lambda x: x.ctypes.data_as(C.c_void_p)                   # noqa: E731
        if self.what == "import":
            rc = _raw(eng, "lane_import_instances", eng._h, lanes[self.kd], buf[1], buf[0].shape[0], P(buf[0]), C.c_size_t(buf[0].shape[1]))
        else:
            rc = _raw(eng, "lane_copy_instances", eng._h, lanes[self.ks], lanes[self.kd], buf[0].size, P(buf[0]), P(buf[1]))
        assert rc == 0
        for v in buf:
            if isinstance(v, np.ndarray):
                v.view(np.uint8)[...] = 0xA5                        # the caller reuses its buffers at once

    def same(self):
        return True


def issue(x, which, eng, lanes=None):
    if isinstance(x, Mv):
        x.issue(eng, lanes)
    elif lanes is None:
        x.issue(which, eng)
    else:
        x.issue(which, eng, lanes[x.lane if isinstance(x, Proc) else x.k])


def run_twins(a, t, seq, lanes):
    torch.cuda.synchronize()
    for x in seq:
        issue(x, "a", a, lanes)
    for x in seq:
        issue(x, "t", t)
    for ln in lanes:
        a.lane_sync(ln)
    t.sync()
    for j, x in enumerate(seq):
        assert x.same(), f"call {j} ({type(x).__name__} {getattr(x, 'what', '')}) differs from the twin"
    assert full_state(a) == full_state(t)


def import_op(rng, k, bank, windows=WINDOWS):
    """a few bank images into window k, at the image size or a wider stride"""
    i0, m = windows[k][:2]
    cnt = int(rng.integers(1, min(6, m) + 1))
    img = bank[rng.integers(0, bank.shape[0], cnt)]
    if rng.integers(2):
        img = padded(img, img.shape[1] + 16 * int(rng.integers(1, 4)))
    return Mv("import", k, k, (img, i0 + int(rng.integers(m - cnt + 1))))


def copy_op(rng, ks, kd, windows=WINDOWS, most=6):
    """distinct destinations in window kd; sources in window ks, none a destination, some repeated"""
    i0s, ms = windows[ks][:2]
    i0d, md = windows[kd][:2]
    cnt = int(rng.integers(1, most))
    dst = i0d + rng.choice(md, cnt, replace=False)
    src = rng.choice(np.setdiff1d(np.arange(i0s, i0s + ms), dst), cnt)
    return Mv("copy", ks, kd, (src, dst))


def rate_move(kind, rng):
    """a device of the 48 kHz group switches to 44.1 kHz, gets its transmitter restamped, moves into the 44.1 kHz group,
    and its old slot is reset on the 48 kHz lane"""
    s = WINDOWS[1][0] + int(rng.integers(WINDOWS[1][1]))
    d = WINDOWS[0][0] + int(rng.integers(WINDOWS[0][1]))
    return [Cfg("rate", 1, s, (np.array([44100.0], np.float32),)),
            Ctl(kind, 1, "tx", (rng.integers(0, 192, 1), rng.integers(0, 256, (1, 5)).astype(np.uint8), s)),
            Mv("copy", 1, 0, ([s], [d])),
            Ctl(kind, 1, "reset", (s, 1))]


def third_engine(kind, oracle, n=288):
    """images of other devices: their own parameters and topologies, fades armed on 10, 150 and 250, state advanced"""
    r = engine(kind, n, sum(BIG))
    try:
        ws = [(0, 100, 96000.0, 61), (128, 64, 44100.0, 62), (192, 96, 48000.0, 63)]
        configure(r, oracle, kind, ws, armed=[10, 150, 250])
        apply_windows(r, ws, 19)
        r.process_packets_host(np.zeros((n, 96 * 6), np.uint8), 24, [96])
        return r.export_instances()
    finally:
        r.close()


# ---- 1. lane moves on three lanes equal engine-level moves on a twin --------------------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_lane_moves_equal_engine_level_moves(oracle, monkeypatch, kind, cpl):
    """Three phases.  In the first two every lane gets process calls, control, configuration and read calls, and moves:
    imports of images from a third engine and from `a` itself, copies within a lane and between lanes, and a rate switch
    that moves a device into the other group and resets its old slot.  The imported and copied devices carry their own
    topology (their group's rate, or another engine's filters), so the K1 choice goes stale.  The third phase disarms every
    fade, then imports and copies envelope-mode devices in and out, so that the engine's count of envelope-mode instances
    crosses zero in both directions between process calls.  Instances outside every window never change."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    a, t = twins(kind)
    rng = np.random.default_rng(110 + cpl)
    bank = image_bank(kind, rng)
    other = third_engine(kind, oracle)
    try:
        for e in (a, t):
            configure(e, oracle, kind, WINDOWS, armed=[3, 130, 200])
            apply_windows(e, WINDOWS, 5)
        free0 = a.export_instances(*FREE).tobytes()
        lanes = [a.lane_open(i0, m) for i0, m, _, _ in WINDOWS]
        for phase in range(2):
            own = a.export_instances()                               # a checkpoint of a itself, restored into running groups
            seq = []
            for r in range(3):
                for k in rng.permutation(3):
                    i0, m, _, _ = WINDOWS[k]
                    seq.append(Proc(kind, k, i0, m, frames_of(k, r), (24, 16)[(r + k) % 2], (r + k + phase) % 3 == 1, 3000 * phase + 10 * r + k))
                    for _ in range(int(rng.integers(2, 5))):
                        u = rng.random()
                        if u < 0.2:
                            seq.append(import_op(rng, k, other if rng.integers(2) else own))
                        elif u < 0.45:
                            seq.append(copy_op(rng, k, k if rng.random() < 0.4 else int(rng.integers(3))))
                        elif u < 0.6:
                            seq.append(read_op(a, kind, rng, k))
                        elif u < 0.8:
                            seq.append(config_op(kind, rng, k, bank))
                        else:
                            seq.append(control_ops(kind, rng, k))
            at = int(rng.integers(len(seq) + 1))
            seq[at:at] = rate_move(kind, rng)
            run_twins(a, t, seq, lanes)
            assert a.export_instances(*FREE).tobytes() == free0, f"phase {phase}"
        # envelope-mode count through zero and back, by imports and copies only
        seq = [Ctl(kind, k, "fade", (None, fs, i0, m)) for k, (i0, m, fs, _) in enumerate(WINDOWS)]
        procs = lambda s: [Proc(kind, k, i0, m, frames_of(k, s), 24, s % 2 == 1, 5000 + 10 * s + k) for k, (i0, m, _, _) in enumerate(WINDOWS)]   # noqa: E731
        seq += procs(0)
        seq += [Mv("import", 1, 1, (other[150:151], 140))] + procs(1)          # 0 -> 1: a fading device connects
        seq += [Mv("copy", 1, 1, ([141], [140]))] + procs(2)                   # 1 -> 0
        seq += [Ctl(kind, 0, "fade", (fade(44100.0, 1, 0.5), 44100.0, 5, 1)), Mv("copy", 0, 2, ([5], [250]))] + procs(3)   # 0 -> 1 -> 2
        seq += [Ctl(kind, 0, "fade", (None, 44100.0, 5, 1)), Mv("copy", 2, 2, ([251], [250]))] + procs(4)                 # 2 -> 1 -> 0
        run_twins(a, t, seq, lanes)
        assert a.export_instances(*FREE).tobytes() == free0
    finally:
        a.close()
        t.close()


# ---- 2. a copy is ordered against both of its lanes and no other -----------------------------------------------------------
class Gate:
    """A host function on a stream that waits for open(), for at most 30 s, and then simply returns."""

    def __init__(self, drv, stream):
        self.flag, entered = threading.Event(), threading.Event()

        @C.CFUNCTYPE(None, C.c_void_p)
        def hold(_):
            entered.set()
            self.flag.wait(30.0)

        self.fn = hold
        assert drv.cuLaunchHostFunc(C.c_void_p(stream), hold, None) == 0
        assert entered.wait(30.0)

    def open(self):
        self.flag.set()


@pytest.mark.parametrize("kind", KINDS)
def test_lane_moves_wait_for_their_lanes_only(oracle, kind):
    """(1) Lane 2 is held: a copy from lane 0 to lane 1 and an import on lane 1 complete while it is.  (2) Lane 0, the
    source, is held behind a process call: the copy into lane 1 does not run, lane 1's stream stays not ready, until the
    gate opens.  (3) Lane 1, the destination, is held: the reset of the copied source on lane 0 waits for the copy, and
    the destination gets the bytes from before the reset.  Then the twin gets every call in issue order."""
    drv = _cuda_driver()
    a, t = twins(kind)
    rng = np.random.default_rng(111)
    other = third_engine(kind, oracle)
    gates = []
    try:
        for e in (a, t):
            configure(e, oracle, kind, WINDOWS, armed=[3, 130])
            apply_windows(e, WINDOWS, 6)
        lanes = [a.lane_open(i0, m) for i0, m, _, _ in WINDOWS]
        stream = lambda k: a.lane_stream(lanes[k])                  # noqa: E731
        # every lane's image staging and instance lists exist before any gate closes
        log = [Mv("import", k, k, (other[WINDOWS[k][0]:WINDOWS[k][0] + 2], WINDOWS[k][0] + 2)) for k in range(3)]
        log += [Mv("copy", (k + 1) % 3, k, ([WINDOWS[(k + 1) % 3][0] + 5], [WINDOWS[k][0] + 7])) for k in range(3)]
        p2 = Proc(kind, 2, 192, 96, BIG[:8], 24, False, 121)
        p0 = Proc(kind, 0, 0, 100, CADENCE, 24, False, 122)
        p1 = Proc(kind, 1, 128, 64, PACED[0], 16, True, 123)
        third = [Mv("copy", 0, 1, ([3, 7, 7], [130, 131, 132])), Mv("import", 1, 1, (other[20:23], 140))]
        source = Mv("copy", 0, 1, ([10, 11], [150, 151]))
        dest = [Mv("copy", 0, 1, ([20], [160])), Ctl(kind, 0, "reset", (20, 1))]
        torch.cuda.synchronize()
        for x in log:
            issue(x, "a", a, lanes)
        for ln in lanes:
            a.lane_sync(ln)

        gates.append(Gate(drv, stream(2)))                           # (1) a third lane held
        issue(p2, "a", a, lanes)
        t0 = time.monotonic()
        for x in third:
            issue(x, "a", a, lanes)
        a.lane_sync(lanes[1])
        a.lane_sync(lanes[0])
        assert not gates[-1].flag.is_set() and time.monotonic() - t0 < 25.0, "a move waited for a third lane"
        assert drv.cuStreamQuery(C.c_void_p(stream(2))) == NOT_READY
        gates[-1].open()
        a.lane_sync(lanes[2])

        gates.append(Gate(drv, stream(0)))                           # (2) the source lane held
        issue(p0, "a", a, lanes)
        issue(source, "a", a, lanes)
        time.sleep(0.3)
        assert drv.cuStreamQuery(C.c_void_p(stream(1))) == NOT_READY, "the copy ran before the source lane's earlier call"
        gates[-1].open()
        a.lane_sync(lanes[1])
        a.lane_sync(lanes[0])

        gates.append(Gate(drv, stream(1)))                           # (3) the destination lane held
        issue(p1, "a", a, lanes)
        for x in dest:
            issue(x, "a", a, lanes)
        time.sleep(0.3)
        assert drv.cuStreamQuery(C.c_void_p(stream(0))) == NOT_READY, "the source lane's reset ran before the copy"
        gates[-1].open()
        for ln in lanes:
            a.lane_sync(ln)

        seq = log + [p2] + third + [p0, source, p1] + dest
        for x in seq:
            issue(x, "t", t)
        t.sync()
        for j, x in enumerate(seq):
            assert x.same(), j
        assert full_state(a) == full_state(t)
        assert a.export_instances(160, 1).tobytes() != a.export_instances(20, 1).tobytes()
    finally:
        for g in gates:
            g.open()
        a.close()
        t.close()


# ---- 3. a device moves to another engine without stopping either farm -------------------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_lane_import_moves_a_group_from_another_engine(oracle, monkeypatch, kind, cpl):
    """Lane 1's window [128, 192) of engine A is exported on the lane between its process calls, brought to the host and
    imported on B's lane over [64, 128) while B's lane 0 keeps processing.  B's next calls on the moved devices give the
    bytes A's give; B's other group and B's whole state equal a twin that did the import as an engine-level call."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    A = engine(kind, 288, sum(BIG))
    B, Bt = engine(kind, 192, sum(BIG)), engine(kind, 192, sum(BIG))
    try:
        configure(A, oracle, kind, WINDOWS, armed=[3, 130, 150])
        apply_windows(A, WINDOWS, 7)
        bw = [(0, 64, 44100.0, 21), (64, 128, 48000.0, 22)]
        for e in (B, Bt):
            configure(e, oracle, kind, bw, armed=[5, 70])
            apply_windows(e, bw, 8)
        la = [A.lane_open(i0, m) for i0, m, _, _ in WINDOWS]
        lb = [B.lane_open(i0, m) for i0, m, _, _ in bw]
        size = A.instance_image_size()
        imgs = torch.full((64 * (size + 32),), SENT, dtype=torch.uint8, device="cuda")
        before = Proc(kind, 1, 128, 64, PACED[0], 24, False, 131)
        nxt = [Proc(kind, 1, 128, 64, PACED[r % 3], (24, 16)[r % 2], r == 1, 132 + r) for r in range(3)]
        bp = [Proc(kind, 0, 0, 64, CADENCE, (24, 16)[r % 2], r == 2, 140 + r) for r in range(4)]
        torch.cuda.synchronize()
        before.issue("a", A, la[1])
        A.lane_export_instances(la[1], 128, 64, imgs.data_ptr(), size + 32)
        for x in nxt:
            x.issue("a", A, la[1])
        A.lane_sync(la[1])
        host = imgs.cpu().numpy().reshape(64, size + 32)
        for x in bp[:2]:
            x.issue("a", B, lb[0])
        B.lane_import_instances(lb[1], host, 64)
        for x in bp[2:]:
            x.issue("a", B, lb[0])
        for x in nxt:
            x.inst0 = 64
            x.issue("t", B, lb[1])
        for ln in lb:
            B.lane_sync(ln)
        for j, x in enumerate(nxt):
            assert x.same(), f"process call {j} after the move"
        for x in bp[:2]:
            x.issue("t", Bt)
        Bt.import_instances(host, inst0=64)
        for x in bp[2:]:
            x.issue("t", Bt)
        for x in nxt:
            x.out["t"] = tuple(torch.zeros_like(v) if v is not None else None for v in x.out["t"])
            x.issue("t", Bt)
        Bt.sync()
        for x in bp + nxt:
            assert x.same()
        assert full_state(B) == full_state(Bt)
    finally:
        A.close()
        B.close()
        Bt.close()


# ---- 4. imports across staging chunks, more uploads in flight than the ring holds, caller buffers reused -------------------
@pytest.mark.parametrize("kind", KINDS)
def test_lane_moves_across_chunks_and_the_ring(oracle, monkeypatch, kind):
    """With 1 MiB staging chunks, a lane import over a 384-instance window at a stride wider than the image crosses several
    chunks, more than the ring's 8 buffers.  Then 14 imports and copies follow on the same lane with no synchronisation.
    The caller's images and lists are overwritten as soon as each call returns."""
    monkeypatch.setenv("DSPI_HOST_CHUNK_MB", "1")
    n = 448
    ws = [(0, 64, 44100.0, 31), (64, 384, 48000.0, 32)]
    a, t = engine(kind, n, 96), engine(kind, n, 96)
    rng = np.random.default_rng(112)
    other = third_engine(kind, oracle, n)
    try:
        for e in (a, t):
            configure(e, oracle, kind, ws, armed=[10, 100, 300])
            apply_windows(e, ws, 9)
        size = a.instance_image_size()
        assert 384 > 3 * ((1 << 20) // size), "the window fits in three chunks"
        lanes = [a.lane_open(i0, m) for i0, m, _, _ in ws]
        seq = [Mv("import", 1, 1, (padded(other[64:448], size + 48), 64), raw=True), Proc(kind, 1, 64, 384, [48, 48], 24, True, 150)]
        for j in range(14):
            if j % 2:
                x = import_op(rng, 1, other, ws)
            else:
                x = copy_op(rng, int(rng.integers(2)), 1, ws, most=40)
            x.raw = True
            seq.append(x)
        seq.append(Proc(kind, 1, 64, 384, [48, 48], 16, False, 151))
        seq.append(Proc(kind, 0, 0, 64, [48, 48], 24, False, 152))
        run_twins(a, t, seq, lanes)
    finally:
        a.close()
        t.close()


# ---- 5. refusals change nothing; engine-level moves with lanes open ---------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_lane_move_refusals_change_nothing(oracle, kind):
    """Unknown and closed lanes, window violations, duplicate or overlapping lists, NULL arguments, a short stride and bad
    image headers (magic, version, arith, band count, size) are refused with no launch and no change.  Then engine-level
    copies and imports with lanes open add the launches they add on an engine without lanes."""
    n, fs = 288, 48000.0
    a, t = engine(kind, n, 256), engine(kind, n, 256)
    try:
        for e in (a, t):
            configure(e, oracle, kind, [(0, n, fs, 31)], armed=[5, 70])
            apply_windows(e, [(0, n, fs, 31)], 8)
        h = a._h
        ok = a.lane_open(64, 100)                                     # window [64, 164)
        ok2 = a.lane_open(192, 64)                                    # window [192, 256)
        closed = a.lane_open(256, 32)
        a.lane_close(closed)
        size = a.instance_image_size()
        good = padded(t.export_instances(0, 4), size + 16)
        P = lambda x: x.ctypes.data_as(C.c_void_p)                    # noqa: E731
        other = engine("q28" if kind != "q28" else "f32f", 64, 64)
        try:
            other_arith = int(other.export_instances(0, 1)[0, 8:12].view(np.uint32)[0])
        finally:
            other.close()

        def imp(ln, inst0, img=good, cnt=None, stride=None, ptr=True):
            cnt = img.shape[0] if cnt is None else cnt
            return _raw(a, "lane_import_instances", h, ln, inst0, cnt, P(img) if ptr else None, C.c_size_t(img.shape[1] if stride is None else stride))

        def cpy(ls, ld, src, dst, sp=True, dp=True):
            s, d = np.asarray(src, np.uint32), np.asarray(dst, np.uint32)
            return _raw(a, "lane_copy_instances", h, ls, ld, s.size, P(s) if sp else None, P(d) if dp else None)

        l0 = a.launch_count
        for ln in (closed, 16, 0xFFFFFFFF):
            assert imp(ln, 64) == EINVAL
            assert cpy(ln, ok, [70], [200]) == EINVAL and cpy(ok, ln, [70], [200]) == EINVAL and cpy(ln, ln, [70], [71]) == EINVAL
        for inst0 in (62, 161, 286, 0xFFFFFFFE):
            assert imp(ok, inst0) == ERANGE, inst0
        for src, dst in (([63], [200]), ([164], [200]), ([70], [191]), ([70], [256]), ([70, 200], [201, 202]), ([70], [288]),
                         ([0xFFFFFFFF], [200]), ([200], [70])):
            assert cpy(ok, ok2, src, dst) == ERANGE, (src, dst)
        assert cpy(ok, ok, [70], [200]) == ERANGE                     # within one lane: dst outside its window
        for src, dst in (([70, 71], [80, 80]), ([70, 80], [80, 90]), ([70, 71], [90, 70])):
            assert cpy(ok, ok, src, dst) == EINVAL, (src, dst)          # a duplicate dst, an index both source and destination
        assert cpy(ok, ok2, [70, 71], [200, 200]) == EINVAL
        assert cpy(ok, ok2, [70], [200], sp=False) == EINVAL and cpy(ok, ok2, [70], [200], dp=False) == EINVAL
        assert imp(ok, 64, ptr=False) == EINVAL and imp(ok, 64, stride=size - 16) == EINVAL
        bands = int(good[0, 12:16].view(np.uint32)[0])
        for off, val in ((0, 0x12345678), (4, 7), (8, other_arith), (12, bands - 1), (16, size + 16)):   # magic, version, arith, bands, size
            bad = good.copy()
            bad[3, off:off + 4] = np.frombuffer(np.uint32(val).tobytes(), np.uint8)
            assert imp(ok, 64, bad) == EINVAL, off
        assert imp(ok, 100, cnt=0) == 0 and cpy(ok, ok2, [], []) == 0
        assert a.launch_count == l0
        a.sync()
        assert full_state(a) == full_state(t)
        # engine-level copies and imports with lanes open issue what they issue on an engine without lanes
        a.lane_import_instances(ok, good, 100)
        a.lane_copy_instances(ok, ok2, [66, 67, 67], [210, 211, 212])
        t.import_instances(good, inst0=100)
        t.copy_instances([66, 67, 67], [210, 211, 212])
        a.sync()
        t.sync()
        calls = [lambda e: e.copy_instances([5, 6, 6], [40, 41, 42]),
                 lambda e: e.import_instances(good, inst0=120),
                 lambda e: e.copy_instances([70], [230]),
                 lambda e: e.import_instances(good[:1], inst0=270)]
        for f in calls:
            counts = []
            for e in (t, a):
                c0 = e.launch_count
                f(e)
                counts.append(e.launch_count - c0)
            assert counts[0] == counts[1]
        for ln in (ok, ok2):
            a.lane_close(ln)
        assert full_state(a) == full_state(t)
    finally:
        a.close()
        t.close()
