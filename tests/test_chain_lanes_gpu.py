"""GPU: lanes, dspi_chain(q)_lane_* - range calls of several clock groups issued on issue queues of their own, which run
side by side.  The bar is a twin engine that gets the same calls, in the same order, as range calls on its engine stream:
every output buffer, the instance images of every instance, the state blob, the S/PDIF transmitters, the preset-mute
envelopes and the configuration records must be byte-identical.  A few instances are also run through the oracle.
Float engines run in both K1 geometries: 288 instances are 32 mod 64, so in the register-pair geometry (DSPI_F32_CPL=2)
lanes share 64-row K1 groups across roles."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                                                  # noqa: E402
from tests.bulk_cases import wire_packet                                                 # noqa: E402
from tests.chain_cases import pcm_bytes                                                  # noqa: E402
from tests.orc import arm_mute_envelope, make_orc_chain, make_orc_chain_q28             # noqa: E402
from tests.test_chain_packets_gpu import orc_run_packets                                 # noqa: E402
from tests.test_chain_ranges_gpu import CASES, KINDS, arm, engine, is_q, pairs, params   # noqa: E402

EINVAL, ERANGE = -22, -34
CADENCE = [44] * 9 + [45]                                   # 44.1 kHz: 441 frames every 10 ms
PACED = [[48, 49, 48, 47, 48], [49, 48, 48], [47, 48, 49, 48]]   # feedback-paced 48 kHz
BIG = [96] * 96                                             # 96 packets of 96 frames


@pytest.fixture
def libm(oracle):
    oracle.set_libm_f64(1)
    yield oracle
    oracle.set_libm_f64(0)


class Proc:
    """One process call over [inst0, inst0 + n): issued on lane `lane` of engine a and as a range call on engine t.  Its
    inputs and both engines' output buffers are allocated before anything is issued (engine streams do not wait for the
    stream torch allocates on)."""

    def __init__(self, kind, lane, inst0, n, frames, bd, sub, seed, pdm=True, status=True):
        self.lane, self.inst0, self.n, self.frames, self.bd, self.sub = lane, inst0, n, list(frames), bd, sub
        F = sum(frames)
        self.pcm_np = pcm_bytes(n, F, bd, seed)
        self.pcm = torch.from_numpy(self.pcm_np).cuda()
        st = (api.ChainEngineQ28 if is_q(kind) else api.ChainEngine)._STATUS.itemsize

        def outs():
            return (torch.zeros((n, pairs(kind), F, 4 if sub else 2), dtype=torch.int32, device="cuda"),
                    torch.zeros((n, F, 8), dtype=torch.int32, device="cuda") if pdm else None,
                    torch.zeros((n, st), dtype=torch.uint8, device="cuda") if status else None)
        self.out = {"a": outs(), "t": outs()}

    def issue(self, which, eng, lane_id=None):
        sp, pd, st = self.out[which]
        ptrs = (sp.data_ptr(), pd.data_ptr() if pd is not None else 0, st.data_ptr() if st is not None else 0)
        form = "subframes" if self.sub else "packets"
        if lane_id is None:
            getattr(eng, "process_%s_range_device" % form)(self.inst0, self.n, self.pcm.data_ptr(), self.bd, self.frames, *ptrs)
        else:
            getattr(eng, "lane_process_%s_device" % form)(lane_id, self.inst0, self.n, self.pcm.data_ptr(), self.bd, self.frames, *ptrs)

    def same(self):
        return all((x is None and y is None) or torch.equal(x, y) for x, y in zip(self.out["a"], self.out["t"]))


def state(eng):
    """everything a later call depends on, and what the getters report"""
    n = eng.n_instances
    w, h, res = eng.collect_bulk_device()
    return (eng.export_instances().tobytes(), eng.state_export().tobytes(), eng.get_spdif_tx().tobytes(), eng.get_preset_mute().tobytes(),
            w.tobytes(), h.tobytes(), res.tobytes(), n)


def configure(eng, oracle, kind, windows, armed):
    """each window at its own rate; preset-mute fades armed on `armed`; random transmitters"""
    chains = {}
    for inst0, n, fs, seed in windows:
        P, bq = params(oracle, kind, n, fs, seed)
        eng.set_params(P, inst0=inst0)
        eng.upload_biquads(bq, inst0=inst0)
        chains[inst0] = (P, bq, fs)
    for i in armed:
        fs = [w[2] for w in windows if w[0] <= i < w[0] + w[1]][0]
        arm(eng, [i], fs)
    rng = np.random.default_rng(eng.n_instances)
    eng.set_spdif_tx(rng.integers(0, 192, eng.n_instances), rng.integers(0, 256, (eng.n_instances, 5)).astype(np.uint8))
    return chains


# ---- 1. three clock groups on three lanes -------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cpl", CASES)
def test_three_lanes_equal_sequential_range_calls(libm, monkeypatch, kind, cpl):
    """A 44.1 kHz group [0, 100) (n not a multiple of 64), a feedback-paced 48 kHz group at the next 64-instance boundary
    [128, 192) with preset-mute fades, and a 96 x 96-frame group [192, 288), three rounds issued interleaved without a host
    synchronisation, with sub-range calls inside a window.  The big group's first call grows the envelope table while
    the other lanes have work queued."""
    monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
    n = 288
    windows = [(0, 100, 44100.0, 11), (128, 64, 48000.0, 12), (192, 96, 96000.0, 13)]
    armed = [3, 130, 131, 150, 200]
    a, t = engine(kind, n, sum(BIG)), engine(kind, n, sum(BIG))
    try:
        cfg = configure(a, libm, kind, windows, armed)
        configure(t, libm, kind, windows, armed)
        mk = make_orc_chain_q28 if is_q(kind) else make_orc_chain
        orc = {}
        for i in (5, 130, 200):
            i0 = max(w for w in cfg if w <= i)
            P, bq, fs = cfg[i0]
            orc[i] = mk(libm, P[i - i0], bq[i - i0])
            if i in armed:
                arm_mute_envelope(orc[i], fs)
        lanes = [a.lane_open(i0, m) for i0, m, _, _ in windows]
        calls = []
        for r in range(3):
            bd, sub = (24, 16, 24)[r], r == 1
            calls += [Proc(kind, 0, 0, 100, CADENCE, bd, sub, 100 + r),
                      Proc(kind, 1, 128, 64, PACED[r], 40 - bd, not sub, 200 + r),
                      Proc(kind, 2, 192, 96, BIG, bd, r == 2, 300 + r, status=r != 1)]
            if r == 1:                                       # sub-ranges inside the windows
                calls += [Proc(kind, 2, 256, 32, BIG[:7], 16, False, 400), Proc(kind, 0, 64, 36, CADENCE, 24, True, 401, pdm=False)]
        torch.cuda.synchronize()
        for p in calls:
            p.issue("a", a, lanes[p.lane])
        for p in calls:
            p.issue("t", t)
        for ln in lanes:
            a.lane_sync(ln)
        t.sync()
        for k, p in enumerate(calls):
            assert p.same(), f"call {k}: lane [{p.inst0}, {p.inst0 + p.n}) differs from the range call"
        assert state(a) == state(t)
        for k, p in enumerate(calls):                        # the oracle, call by call, on a few instances
            for i, ch in orc.items():
                if p.inst0 <= i < p.inst0 + p.n:
                    ws, wp = orc_run_packets(libm, kind, ch, p.pcm_np[i - p.inst0], p.bd, p.frames)
                    sp, pd, _ = (x.cpu().numpy() if x is not None else None for x in p.out["a"])
                    if not p.sub:
                        assert np.array_equal(sp[i - p.inst0], ws), f"call {k} instance {i}: S/PDIF words differ from the oracle"
                    if pd is not None and int(ch.out[4 if is_q(kind) else 8].enabled):
                        assert np.array_equal(pd[i - p.inst0].view(np.uint32), wp), f"call {k} instance {i}: PDM differs from the oracle"
    finally:
        a.close()                                            # destroyed with its lanes open
        t.close()


# ---- 2. engine-level calls are barriers ---------------------------------------------------------------------------------
def _packets(eng, n, seed):
    return np.concatenate([wire_packet(eng._PLATFORM, seed + i) for i in range(n)])


@pytest.mark.parametrize("kind", KINDS)
def test_engine_level_calls_between_lane_calls(oracle, kind):
    """Lane calls interleaved with apply / edit / copy / rate switch / reset / transmitter / whole-engine process /
    response calls, no host synchronisation in between; a lane closed with work queued and reopened; dspi_chain_sync
    waits for the lanes."""
    n, fs = 160, 48000.0
    wa, wb = (0, 64), (64, 96)
    a, t = engine(kind, n, 1024), engine(kind, n, 1024)
    try:
        for e in (a, t):
            configure(e, oracle, kind, [(0, n, fs, 21)], armed=[2, 70])
        packets = _packets(a, n, 900)
        edits = np.concatenate([L.bulk_edit(3, ("outputs", 0, "gain_db"), np.float32(-6.0)), L.bulk_edit(90, ("host", "volume_8_8"), -9 * 256),
                                L.bulk_edit(64, ("crossfeed", "enabled"), 1)])
        freqs = np.array([50.0, 1000.0, 15000.0], np.float32)
        resp = {w: torch.zeros((n, a._OUTS, 2, 3, 2), dtype=torch.float32, device="cuda") for w in "at"}
        whole = Proc(kind, None, 0, n, [96, 96], 24, False, 77)
        rounds = [[Proc(kind, 0, 0, 64, CADENCE, 24, False, 500 + r), Proc(kind, 1, 64, 96, PACED[r % 3], 16, r % 2 == 1, 600 + r)] for r in range(7)]
        moved = Proc(kind, 1, 64, 32, [48] * 3, 24, False, 700)                 # serves the copied device in its new window
        late = Proc(kind, 1, 64, 96, [96], 24, False, 701)
        torch.cuda.synchronize()
        results = {}
        for w, e in (("a", a), ("t", t)):
            ids = [a.lane_open(*wa), a.lane_open(*wb)] if w == "a" else [None, None]
            lane = lambda k: ids[k]                                           # noqa: E731
            res = []
            run = lambda r: [p.issue(w, e, lane(p.lane)) for p in rounds[r]]  # noqa: E731
            run(0)
            res.append(e.apply_bulk_device(packets, fs))
            run(1)
            res.append(e.edit_bulk_device(edits, fs))
            run(2)
            e.copy_instances([5], [70])                                       # a device moved from one window to the other
            moved.issue(w, e, lane(1))
            res.append(e.set_rate_device(np.full(96, 44100.0, np.float32), inst0=64))
            run(3)
            e.reset_instances(10, 5)
            e.set_spdif_tx(17, np.arange(5, dtype=np.uint8), inst0=100)
            run(4)
            whole.issue(w, e)                                                 # a whole-engine range call on the engine stream
            e.response(freqs, fs, out_ptr=resp[w].data_ptr())
            run(5)
            if w == "a":                                                      # close with work queued, then reopen
                a.lane_close(ids[1])
                ids[1] = a.lane_open(*wb)
            run(6)
            late.issue(w, e, lane(1))
            e.sync()                                                          # waits for the lanes too
            results[w] = res
        for x, y in zip(results["a"], results["t"]):
            assert np.array_equal(x, y)
        assert torch.equal(resp["a"], resp["t"])
        for k, p in enumerate([q for r in rounds for q in r] + [moved, late, whole]):
            assert p.same(), f"call {k}"
        assert state(a) == state(t)
    finally:
        a.close()
        t.close()


# ---- 3. refusals change nothing; no lane open, no extra work -----------------------------------------------------------
def _raw(eng, name, *args):
    return getattr(api.lib(), eng._PRE + "_" + name)(*args)


@pytest.mark.parametrize("kind", KINDS)
def test_lane_refusals_change_nothing(oracle, kind):
    n, fs, F = 1100, 48000.0, 96
    a, t = engine(kind, n, 256), engine(kind, n, 256)
    try:
        for e in (a, t):
            configure(e, oracle, kind, [(0, n, fs, 31)], armed=range(0, n, 50))
            e.process_packets_host(pcm_bytes(n, F, 24, 72), 24, [F])
        h = a._h
        lane = C.c_uint32(99)
        ok = a.lane_open(64, 100)
        assert _raw(a, "lane_open", h, 0, 64, None) == EINVAL                         # NULL lane pointer
        for inst0, m, rc in ((32, 64, EINVAL), (0, 0, EINVAL), (128, 64, EINVAL), (0, 65, EINVAL), (1088, 64, ERANGE), (1024, 77, ERANGE),
                             (0xFFFFFFC0, 0x80, ERANGE)):
            assert _raw(a, "lane_open", h, inst0, m, C.byref(lane)) == rc, (inst0, m)
        assert lane.value == 99
        extra = [a.lane_open(192 + 64 * k, 64) for k in range(14)] + [a.lane_open(1088, 12)]   # 16 lanes open
        assert _raw(a, "lane_open", h, 0, 64, C.byref(lane)) == ERANGE                  # a 17th
        assert lane.value == 99
        pcm = torch.from_numpy(pcm_bytes(n, F, 24, 73)).cuda()
        sp = torch.full((n * pairs(kind) * F * 4 + 4,), 7, dtype=torch.int32, device="cuda")
        pd = torch.full((n, F, 8), 7, dtype=torch.int32, device="cuda")
        st = torch.full((n, 64), 7, dtype=torch.uint8, device="cuda")
        sp0, pd0, st0 = sp.clone(), pd.clone(), st.clone()
        tab = np.array([F, 0], np.uint16)
        p = C.c_void_p(pcm.data_ptr())
        outs = (C.c_void_p(sp.data_ptr()), C.c_void_p(pd.data_ptr()), C.c_void_p(st.data_ptr()))
        torch.cuda.synchronize()

        def both(ln, inst0, m, p=p, nk=1, table=tab.ctypes.data, bd=24):
            return tuple(_raw(a, "lane_process_%s_device" % form, h, ln, inst0, m, p, bd, nk, table, *outs) for form in ("packets", "subframes"))

        closed = extra.pop()
        a.lane_close(closed)
        assert a.lane_stream(closed) is None and a.lane_stream(ok) is not None
        assert both(closed, 1024, 10) == (EINVAL, EINVAL)                              # closed lane
        assert both(16, 64, 10) == (EINVAL, EINVAL)                                    # unknown lane
        assert both(ok, 32, 10) == (EINVAL, EINVAL)                                    # misaligned
        assert both(ok, 64, 101) == (ERANGE, ERANGE)                                   # past the window
        assert both(ok, 128, 64) == (ERANGE, ERANGE)
        assert both(ok, 0, 64) == (ERANGE, ERANGE)                                     # before the window
        assert both(ok, 1088, 64) == (ERANGE, ERANGE)                                  # past the engine
        assert both(ok, 64, 10, p=None) == (EINVAL, EINVAL)
        assert both(ok, 64, 10, nk=2) == (EINVAL, EINVAL)                              # a packet of 0 frames
        assert both(ok, 64, 10, nk=0) == (EINVAL, EINVAL)
        assert both(ok, 64, 10, table=None) == (EINVAL, EINVAL)
        assert both(ok, 64, 10, bd=20) == (EINVAL, EINVAL)
        assert _raw(a, "lane_process_subframes_device", h, ok, 64, 10, p, 24, 1, tab.ctypes.data, C.c_void_p(sp.data_ptr() + 4), *outs[1:]) == EINVAL
        assert _raw(a, "lane_close", h, closed) == EINVAL and _raw(a, "lane_sync", h, 16) == EINVAL
        l0 = a.launch_count
        assert both(ok, 128, 0) == (0, 0)                                              # n == 0 does nothing
        assert a.launch_count == l0
        a.sync()
        assert torch.equal(sp, sp0) and torch.equal(pd, pd0) and torch.equal(st, st0)
        assert state(a) == state(t)
        # with every lane closed again, an engine call issues what it issued before any lane was opened
        for ln in extra + [ok]:
            a.lane_close(ln)
        pcm_np = pcm_bytes(n, F, 24, 74)
        counts = []
        for e in (t, a):
            l0 = e.launch_count
            e.process_packets_host(pcm_np, 24, [48, 48])
            counts.append(e.launch_count - l0)
        assert counts[0] == counts[1]
        assert state(a) == state(t)
    finally:
        a.close()
        t.close()
