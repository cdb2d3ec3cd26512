"""GPU: lane host calls, dspi_chain(q)_lane_process_packets_host / _lane_process_subframes_host - a clock group's packets
served from page-locked host memory on its lane, each packet slice copied in and out while the stages run, without a host
synchronisation.  The bar is a twin engine that gets the same calls in the same order, the lane host calls as engine-level
range host calls (process_*_range_host), the lane device and control calls as their engine-level forms: every output
(words, subframes, PDM, status), the state blob, the transmitters, the envelopes and the configuration records must be
byte-identical.  Float engines run in both K1 geometries."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                                  # noqa: E402
from tests.chain_cases import pcm_bytes                                                  # noqa: E402
from tests.test_chain_lane_control_gpu import (WINDOWS, Ctl, _cuda_driver, _raw, apply_windows, control_ops, frames_of,   # noqa: E402
                                               full_state)
from tests.test_chain_lanes_gpu import BIG, CADENCE, PACED, Proc, configure              # noqa: E402
from tests.test_chain_ranges_gpu import CASES, KINDS, engine, is_q, pairs                # noqa: E402

EINVAL, ERANGE = -22, -34
SENT = 0x5A


def sub_of(kind):
    return 2 * pairs(kind)                                   # the sub output: after the S/PDIF pairs


class HProc:
    """One host process call over [inst0, inst0 + n): issued on lane `lane` of engine a from pinned buffers prefilled with
    SENT, and as the engine-level range host call on engine t (which returns numpy arrays)."""

    def __init__(self, kind, lane, inst0, n, frames, bd, sub, seed, spdif=True, pdm=True, status=True):
        self.lane, self.inst0, self.n, self.frames, self.bd, self.sub = lane, inst0, n, list(frames), bd, sub
        self.want = (spdif, pdm, status)
        F = sum(frames)
        self.pcm_np = pcm_bytes(n, F, bd, seed)
        self.pcm = torch.from_numpy(self.pcm_np).pin_memory()
        st = (api.ChainEngineQ28 if is_q(kind) else api.ChainEngine)._STATUS.itemsize
        shapes = ((n, pairs(kind), F, 4 if sub else 2), (n, F, 8), (n, st))
        self.out = [torch.full(s, SENT if j == 2 else SENT * 0x01010101, dtype=torch.uint8 if j == 2 else torch.int32).pin_memory() if w else None
                    for j, (s, w) in enumerate(zip(shapes, self.want))]
        self.ref = None

    def issue(self, which, eng, lane_id=None):
        if lane_id is None:
            form = "subframes" if self.sub else "packets"
            self.ref = getattr(eng, "process_%s_range_host" % form)(self.inst0, self.pcm_np, self.bd, self.frames, *self.want)
            return
        eng.lane_process_packets_host(lane_id, self.inst0, self.pcm, self.bd, self.frames, *self.out, subframes=self.sub)

    def got(self):
        return [x.numpy().tobytes() if x is not None else None for x in self.out]

    def same(self):
        return all((g is None and r is None) or (r is not None and g == np.ascontiguousarray(r).tobytes()) for g, r in zip(self.got(), self.ref))


def run(eng, which, seq, lanes=None):
    for x in seq:
        k = x.lane if isinstance(x, (Proc, HProc)) else x.k
        x.issue(which, eng, None if lanes is None or k is None else lanes[k])


def sub_off(kind, k, insts):
    """a Console switching the sub of some instances of window k off"""
    return Ctl(kind, k, "edit", (np.concatenate([L.bulk_edit(i, ("outputs", sub_of(kind), "enabled"), 0) for i in insts]), WINDOWS[k][2]))


# ---- 1. host calls on three lanes equal engine-level range host calls on a twin ---------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_lane_host_calls_equal_range_host_calls(oracle, monkeypatch, kind, cpl):
    """Three phases; in each, every lane gets host calls (16- and 24-bit, words and subframes, the 44.1 kHz cadence, paced
    tables, one-packet calls, a max_frames call of 16 slices on the 96-instance window; window 0 has n = 100), device calls,
    control calls and an engine-level call, interleaved across the lanes without a host synchronisation.  Between phases a
    Console switches subs off, and the host calls after it must return those PDM rows as zeros."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    a, t = engine(kind, 288, sum(BIG)), engine(kind, 288, sum(BIG))
    rng = np.random.default_rng(60 + cpl)
    try:
        for e in (a, t):
            configure(e, oracle, kind, WINDOWS, armed=[3, 130, 200])
            apply_windows(e, WINDOWS, 5)
        lanes = [a.lane_open(i0, m) for i0, m, _, _ in WINDOWS]
        offs = [[5, 6, 97], [130], [192, 250]]
        for phase in range(3):
            seq = []
            for r in range(3):
                for k in rng.permutation(3):
                    i0, m, _, _ = WINDOWS[k]
                    bd, sub, seed = (24, 16)[(r + k) % 2], (r + k + phase) % 3 == 1, 1000 * phase + 10 * r + k
                    frames = [48] if (r + phase) % 3 == 2 else BIG if (k == 2 and r == phase) else frames_of(k, r)
                    outs = [(True, True, True), (True, False, True), (False, True, False)][(r + k) % 3] if r == 1 else (True, True, True)
                    seq.append(HProc(kind, k, i0, m, frames, bd, sub, seed, *outs))
                    u = rng.random()
                    if u < 0.3:
                        seq.append(Proc(kind, k, i0, m, frames_of(k, r + 1), 40 - bd, not sub, seed + 500))
                    elif u < 0.7:
                        seq.append(control_ops(kind, rng, k))
                if r == 1:                                                  # an engine-level call: a barrier across lanes
                    seq.append(Proc(kind, None, 0, 288, [96, 96], 24, phase == 1, 3000 + phase))
                    seq.append(HProc(kind, 0, 64, 36, CADENCE, 24, False, 3100 + phase))   # a sub-range inside window 0
            if phase == 1:
                for k in range(3):
                    seq.append(sub_off(kind, k, offs[k]))
                seq += [HProc(kind, k, WINDOWS[k][0], WINDOWS[k][1], frames_of(k, 0), 24, k == 1, 3200 + k) for k in range(3)]
            torch.cuda.synchronize()
            run(a, "a", seq, lanes)
            run(t, "t", seq)
            for ln in lanes:
                a.lane_sync(ln)
            t.sync()
            for j, x in enumerate(seq):
                assert x.same(), f"phase {phase}, call {j} ({type(x).__name__} {getattr(x, 'what', '')}) differs from the twin"
            assert full_state(a) == full_state(t), f"phase {phase}"
            if phase == 1:
                for x in seq[-3:]:
                    pdm = x.out[1].numpy()
                    for i in offs[x.lane]:
                        assert not pdm[i - x.inst0].any(), f"instance {i}: PDM of a sub switched off is not zero"
    finally:
        a.close()
        t.close()


# ---- 2. a host call does not wait, and does not hold the other lanes --------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_lane_host_calls_do_not_wait(oracle, kind):
    """Lane 0's stream is held by a host gate (a host function that waits for a flag, for at most 30 s, and then simply
    returns).  A host call on lane 0 returns and its stream reports not ready; host calls on lane 1 complete meanwhile.
    Then the gate opens and every result equals the twin's."""
    drv = _cuda_driver()
    a, t = engine(kind, 288, sum(BIG)), engine(kind, 288, sum(BIG))
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
        warm = [HProc(kind, k, WINDOWS[k][0], WINDOWS[k][1], frames_of(k, 0), 24, sub, 70 + k + 2 * sub) for k in range(2) for sub in (False, True)]
        held = HProc(kind, 0, 0, 100, CADENCE, 24, False, 75)
        other = [HProc(kind, 1, 128, 64, PACED[r], (24, 16)[r % 2], r == 1, 76 + r) for r in range(3)]
        torch.cuda.synchronize()
        run(a, "a", warm, lanes)                                      # every staging exists before the gate closes
        for ln in lanes:
            a.lane_sync(ln)
        s0 = C.c_void_p(a.lane_stream(lanes[0]))
        assert drv.cuLaunchHostFunc(s0, hold, None) == 0
        assert entered.wait(30.0)
        t0 = time.monotonic()
        run(a, "a", [held], lanes)
        assert drv.cuStreamQuery(s0) == 600, "lane 0 reports ready while held"   # CUDA_ERROR_NOT_READY
        run(a, "a", other, lanes)
        a.lane_sync(lanes[1])
        assert not gate.is_set() and time.monotonic() - t0 < 25.0, "a lane host call waited for the held lane 0"
        assert drv.cuStreamQuery(s0) == 600
        gate.set()
        a.lane_sync(lanes[0])
        run(t, "t", warm + [held] + other)
        for j, x in enumerate(warm + [held] + other):
            assert x.same(), j
        assert full_state(a) == full_state(t)
    finally:
        gate.set()
        a.close()
        t.close()


# ---- 3. pcm is read on the lane's timeline ----------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_lane_host_pcm_is_reused_after_the_lane_reaches_the_call(oracle, kind):
    """One pinned PCM buffer and one set of pinned outputs serve five calls of a group; each is rewritten only after the
    lane has reached the end of the previous call, shown by an event recorded on the lane stream (or by lane_sync)."""
    a, t = engine(kind, 288, 1024), engine(kind, 288, 1024)
    try:
        for e in (a, t):
            configure(e, oracle, kind, WINDOWS, armed=[130])
        lane = a.lane_open(128, 64)
        tables = [PACED[0], [48] * 5, [96, 96, 48], [120, 120], [47, 49, 48, 48, 48]]       # 240 frames each
        x = HProc(kind, 1, 128, 64, tables[0], 24, False, 80)
        stream = torch.cuda.ExternalStream(a.lane_stream(lane))
        for r, frames in enumerate(tables):
            x.frames = frames
            x.pcm_np = pcm_bytes(64, sum(frames), 24, 81 + r)
            x.pcm.numpy()[...] = x.pcm_np                            # the previous call has been read: rewrite
            x.issue("a", a, lane)
            if r % 2:
                a.lane_sync(lane)
            else:
                ev = torch.cuda.Event()
                ev.record(stream)
                ev.synchronize()
            x.issue("t", t)
            assert x.same(), f"call {r}"
        assert full_state(a) == full_state(t)
    finally:
        a.close()
        t.close()


# ---- 4. refusals change nothing ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_lane_host_refusals_change_nothing(oracle, kind):
    n, fs, F = 288, 48000.0, 96
    a, t = engine(kind, n, 256), engine(kind, n, 256)
    try:
        for e in (a, t):
            configure(e, oracle, kind, [(0, n, fs, 31)], armed=[5, 70])
        h = a._h
        ok = a.lane_open(64, 100)                                     # window [64, 164)
        closed = a.lane_open(192, 64)
        a.lane_close(closed)
        st = a._STATUS.itemsize
        pcm = torch.from_numpy(pcm_bytes(100, F, 24, 90)).pin_memory()
        sp = torch.full((100 * pairs(kind) * F * 4,), 7, dtype=torch.int32).pin_memory()
        pd = torch.full((100, F, 8), 7, dtype=torch.int32).pin_memory()
        stt = torch.full((100, st), 7, dtype=torch.uint8).pin_memory()
        pageable = np.full(100 * F * 6 + 64 * pairs(kind) * F * 16, 7, np.uint8)
        dev = torch.full((100 * pairs(kind) * F * 16,), 7, dtype=torch.uint8, device="cuda")
        keep = [x.clone() for x in (sp, pd, stt)]
        tab = np.array([F, 0], np.uint16)
        P = C.c_void_p(pcm.data_ptr())
        outs = (C.c_void_p(sp.data_ptr()), C.c_void_p(pd.data_ptr()), C.c_void_p(stt.data_ptr()))
        pg = C.c_void_p(pageable.ctypes.data)
        before = full_state(a)
        torch.cuda.synchronize()

        def both(ln, inst0, m, p=P, nk=1, table=tab.ctypes.data, bd=24, o=outs):
            return tuple(_raw(a, "lane_process_%s_host" % form, h, ln, inst0, m, p, bd, nk, table, *o) for form in ("packets", "subframes"))

        l0 = a.launch_count
        assert both(closed, 192, 10) == (EINVAL, EINVAL)                               # closed lane
        assert both(16, 64, 10) == (EINVAL, EINVAL)                                    # unknown lane
        assert both(0xFFFFFFFF, 64, 10) == (EINVAL, EINVAL)
        assert both(ok, 32, 10) == (EINVAL, EINVAL)                                    # misaligned
        assert both(ok, 64, 101) == (ERANGE, ERANGE)                                   # past the window
        assert both(ok, 128, 64) == (ERANGE, ERANGE)
        assert both(ok, 0, 64) == (ERANGE, ERANGE)                                     # before the window
        assert both(ok, 0xFFFFFFC0, 0x80) == (ERANGE, ERANGE)                          # wraps in 32 bits
        assert both(ok, 64, 10, p=None) == (EINVAL, EINVAL)
        assert both(ok, 64, 10, nk=2) == (EINVAL, EINVAL)                              # a packet of 0 frames
        assert both(ok, 64, 10, nk=0) == (EINVAL, EINVAL)
        assert both(ok, 64, 10, table=None) == (EINVAL, EINVAL)
        assert both(ok, 64, 10, bd=20) == (EINVAL, EINVAL)
        big = np.array([150, 150], np.uint16)                                          # 300 frames > max_frames 256
        assert both(ok, 64, 10, nk=2, table=big.ctypes.data) == (ERANGE, ERANGE)
        assert both(ok, 64, 10, p=pg) == (EINVAL, EINVAL)                              # pageable pcm
        for j in range(3):                                                             # a pageable or device output
            for bad in (pg, C.c_void_p(dev.data_ptr())):
                o = list(outs)
                o[j] = bad
                assert both(ok, 64, 10, o=tuple(o)) == (EINVAL, EINVAL), j
                assert b"page-locked" in api.lib().dspi_last_error()
        assert both(ok, 64, 10, p=C.c_void_p(dev.data_ptr())) == (EINVAL, EINVAL)      # device pcm
        assert both(ok, 128, 0) == (0, 0)                                              # n == 0 does nothing
        with pytest.raises(api.DspiError):
            a.lane_process_packets_host(ok, 64, torch.from_numpy(pcm_bytes(100, F, 24, 91)), 24, [F])   # not pinned
        assert a.launch_count == l0
        a.sync()
        assert torch.equal(sp, keep[0]) and torch.equal(pd, keep[1]) and torch.equal(stt, keep[2])
        assert (pageable == 7).all() and (dev.cpu() == 7).all()
        assert full_state(a) == before
        # the lane still works, and equals the engine-level range host call
        x = HProc(kind, 0, 64, 100, [F], 24, True, 92)
        x.issue("a", a, ok)
        a.lane_sync(ok)
        x.issue("t", t)
        assert x.same()
        assert full_state(a) == full_state(t)
    finally:
        a.close()
        t.close()
