"""GPU: the leveller's level-dependent paths against the oracle under the libm policy (oracle `libm_f64`, ARM conversions),
bit for bit - gate, boost, knee, compression, max-gain clamp, the peak limiter, the Q28 gain saturation and the Q28
envelope that goes below zero, on the signals whose reach tests/test_leveller_paths_cpu.py counts.

Every instance starts from a settled leveller state (tests/leveller_cases.py) written into the engine through the state
blob and into the oracle's record; after every call the S/PDIF words, PDM bits, peaks, clip flags and the leveller part
of the state blob (both envelopes, smoothed gain, gain and previous gain, the 480-slot look-ahead ring and its index)
must equal the oracle's.  One exception in kind, not in degree: a smoothed gain that is NaN on both sides (Q28 envelope
below zero) is equal whatever its payload, which neither C nor CUDA defines."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from dspi_b200 import api, layouts as L                      # noqa: E402
from tests import leveller_cases as LC                        # noqa: E402
from tests.test_dynamics_gpu import apply_to_oracle           # noqa: E402

CADENCE_44K1 = [44] * 9 + [45]
VARIANTS = [("f32f", 0), ("f32s", 1), ("f32s", 2), ("q28", 0)]
VARIANT_IDS = ["f32f", "f32s-cpl1", "f32s-cpl2", "q28"]


@pytest.fixture(autouse=True)
def _plain_paths(monkeypatch):
    monkeypatch.delenv("DSPI_JIT", raising=False)
    monkeypatch.delenv("DSPI_DBG", raising=False)
    monkeypatch.delenv("DSPI_F32_CPL", raising=False)


def _canon(a):
    """Bit patterns; float NaNs of any payload as one pattern."""
    a = np.ascontiguousarray(a)
    if a.dtype.kind != "f":
        return a.view(np.uint32)
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7FC00000
    return b


class Run:
    """An engine and one oracle instance per engine instance, both started from the instances' settled states; every
    instance consumes its own PCM stream, whatever calls or ranges it is processed in."""

    def __init__(self, monkeypatch, oracle, flavour, insts, P, bq, max_frames, cpl=0):
        self.oracle, self.flavour, self.q28 = oracle, flavour, flavour == "q28"
        self.insts, self.P, self.N = insts, P, len(insts)
        self.bd = insts[0].bit_depth
        self.bpf = 6 if self.bd == 24 else 4
        if cpl:
            monkeypatch.setenv("DSPI_F32_CPL", str(cpl))
        self.eng = api.ChainEngineQ28(self.N, max_frames=max_frames) if self.q28 else api.ChainEngine(flavour, self.N, max_frames=max_frames)
        self.eng.set_params(P)
        self.eng.upload_biquads(bq)
        LC.write_settled(self.eng, self.q28, insts)
        self.chains = [LC.oracle_chain(oracle, self.q28, P[i], bq[i], it) for i, it in enumerate(insts)]
        self.pcm = [LC.pcm_of(it.body, self.bd) for it in insts]
        self.pos = [0] * self.N                         # frames of its stream each instance has consumed
        self.remainders = {1: 0, -1: 0}                 # signs of the Q28 ramp remainder (g_cur - g_prev) % (count - 1)
        self.sub_o = (L.CHAINQ_OUTPUTS if self.q28 else L.CHAIN_OUTPUTS) - 1
        self.state_check(LC.levs_record, "settled state written")

    def close(self):
        self.eng.close()

    def _oracle(self, i, frames):
        """The oracle instance i over the packets `frames`, from where its stream stands; returns (spdif, pdm)."""
        ch, F = self.chains[i], int(sum(frames))
        spdif = np.zeros((2 if self.q28 else 4, F, 2), np.int32)
        pdm = np.zeros((F, 8), np.uint32)
        fn = getattr(self.oracle.lib, f"orc_{self.flavour}_chain_packet")
        data = self.pcm[i]
        f0 = 0
        for n in frames:
            n = int(n)
            g_prev = ch.levs.gain_q28 if self.q28 else 0
            fn(C.addressof(ch), data.ctypes.data + (self.pos[i] + f0) * self.bpf, n * self.bpf, self.bd,
               spdif.ctypes.data + f0 * 8, F * 2, pdm.ctypes.data + f0 * 32)
            if self.q28 and ch.leveller_on and n > 2:
                diff = int(np.int32(np.int64(ch.levs.gain_q28) - g_prev))
                r = (abs(diff) % (n - 1)) * (1 if diff > 0 else -1)
                if r:
                    self.remainders[1 if r > 0 else -1] += 1
            f0 += n
        self.pos[i] += F
        return spdif, pdm

    def call(self, frames, inst0=None, n=None):
        """One process call over the whole engine (inst0 None) or over instances [inst0, inst0 + n), checked against the
        oracle instance by instance."""
        rows = range(self.N) if inst0 is None else range(inst0, inst0 + n)
        F = int(sum(frames))
        chunk = np.ascontiguousarray(np.stack([self.pcm[i][self.pos[i] * self.bpf:(self.pos[i] + F) * self.bpf] for i in rows]))
        if inst0 is None:
            spdif, pdm, status = self.eng.process_packets_host(chunk, self.bd, frames)
        else:
            spdif, pdm, status = self.eng.process_packets_range_host(inst0, chunk, self.bd, frames)
        what = f"call of {len(frames)} packets" + ("" if inst0 is None else f" over [{inst0}, {inst0 + n})")
        for k, i in enumerate(rows):
            ws, wp = self._oracle(i, frames)
            ch, case = self.chains[i], self.insts[i].case
            assert np.array_equal(spdif[k], ws), f"{what}: instance {i} {case}: S/PDIF words differ, first at {np.argwhere(spdif[k] != ws)[0]}"
            if self.P[i]["matrix"]["outputs"][self.sub_o]["enabled"]:
                assert np.array_equal(pdm[k], wp), f"{what}: instance {i} {case}: PDM bits differ"
            n_roles = len(status[k]["peaks"])
            assert list(status[k]["peaks"]) == list(ch.peaks)[:n_roles], f"{what}: instance {i} {case}: peaks"
            assert int(status[k]["clip_flags"]) == int(ch.clip_flags), f"{what}: instance {i} {case}: clip flags"
        self.state_check(LC.levs_record, what)

    def state_check(self, record, what):
        v = LC.blob_leveller(self.eng.state_export(), self.q28, self.N)
        for i, ch in enumerate(self.chains):
            want = record(ch, self.q28)
            for f in want.dtype.names:
                got, exp = _canon(v[f][i]), _canon(want[f][0])
                assert np.array_equal(got, exp), f"{what}: instance {i} {self.insts[i].case}: leveller state '{f}' differs" + \
                    (f" (engine {got.ravel()[:1]}, oracle {exp.ravel()[:1]})" if got.size == 1 else f" at {np.argwhere(got != exp)[:3].tolist()}")


def _split(frames, cuts):
    out, k = [], 0
    for c in list(cuts) + [len(frames)]:
        out.append(frames[k:c])
        k = c
    return out


def _run_calls(monkeypatch, oracle, flavour, insts, P, bq, calls, cpl=0):
    oracle.set_libm_f64(1)
    r = Run(monkeypatch, oracle, flavour, insts, P, bq, max(int(sum(c)) for c in calls), cpl)
    try:
        for frames in calls:
            r.call(frames)
        return r.remainders
    finally:
        r.close()
        oracle.set_libm_f64(0)


# ---- 1. the census's sets, level-controlled and with every stage on ----------------------------------------------------
SETS = {"level24": ("level24", False, [17]), "level16": ("level16", False, [29]), "stages24": ("level24", True, [17])}


@pytest.mark.parametrize("set_name", list(SETS))
@pytest.mark.parametrize("flavour,cpl", VARIANTS, ids=VARIANT_IDS)
def test_leveller_paths_match_the_oracle(monkeypatch, oracle, flavour, cpl, set_name):
    """44 instances (N_pad 64, two warps' worth of instances past the last full one), one call split from the next at an
    arbitrary packet"""
    base, stages, cuts = SETS[set_name]
    n, fs, bd, frames, seed = LC.LEVEL_SETS[base]
    insts, P, bq, _ = LC.make_set(oracle, flavour, n, fs, bd, sum(frames), seed, stages=stages)
    _run_calls(monkeypatch, oracle, flavour, insts, P, bq, _split(frames, cuts), cpl)


# ---- 2. packet schedules -------------------------------------------------------------------------------------------------
def _mixed():
    rng = np.random.default_rng(61)
    return [int(x) for x in rng.choice([1, 2, 3, 44, 45, 47, 95, 96, 191, 192], 40)]


SCHEDULES = {
    "1-frame": (96000.0, [1] * 600, [250]),         # the count == 1 branch (no ramp); 600 frames wrap the ring
    "2-frame": (96000.0, [2] * 300, [131]),
    "47-frame": (96000.0, [47] * 40, [13, 27]),     # the ring wraps inside packets
    "192-frame": (96000.0, [192] * 20, [7]),
    "44k1": (44100.0, CADENCE_44K1 * 4, [23]),       # 44 / 45 frames
    "mixed": (96000.0, _mixed(), [11, 28]),
}


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_leveller_packet_schedules(monkeypatch, oracle, flavour, schedule):
    """24 instances (every anchor case and 8 drawn ones), 24-bit, level set, calls split at arbitrary packets"""
    fs, frames, cuts = SCHEDULES[schedule]
    insts, P, bq, _ = LC.make_set(oracle, flavour, 24, fs, 24, sum(frames), 71)
    rem = _run_calls(monkeypatch, oracle, flavour, insts, P, bq, _split(frames, cuts))
    if flavour == "q28" and max(frames) > 2:
        # the incremental ramp division (chain_q28.cu) has a correction step per sign of the remainder
        assert rem[1] > 0 and rem[-1] > 0, f"ramp remainders reached: {rem}"


# ---- 3. warp shapes ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_leveller_warp_shapes(monkeypatch, oracle, flavour):
    """N = 70 (N_pad 96, not a multiple of 32) with the leveller off on every third instance, so every 16-instance warp
    half holds lanes that walk the leveller path (__any_sync) without committing; range calls over [0, 64) and over the
    6-instance tail [64, 70) - a warp with 6 live lanes - each with its own packet schedule (the range entry points take
    a first instance that is a multiple of 64)."""
    insts, P, bq, _ = LC.make_set(oracle, flavour, 70, 96000.0, 24, 40 * 96, 81)
    P["leveller_enabled"][np.arange(70) % 3 == 1] = 0
    oracle.set_libm_f64(1)
    r = Run(monkeypatch, oracle, flavour, insts, P, bq, 14 * 96)
    try:
        r.call([96] * 9)
        r.call([96] * 14, inst0=0, n=64)
        r.call([47] * 10 + [45] * 3, inst0=64, n=6)
        r.call([1] * 5 + [192] * 3, inst0=64, n=6)
        r.call([158], inst0=64, n=6)                           # the tail catches up: 605 + 581 + 158 = 14 x 96 frames
        assert len(set(r.pos)) == 1
        r.call([96] * 6)
    finally:
        r.close()
        oracle.set_libm_f64(0)


# ---- 4. live reconfiguration ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["f32f", "f32s", "q28"])
def test_leveller_live_reconfiguration(monkeypatch, oracle, flavour):
    """A running engine reconfigured on the device between calls (dspi_chain(q)_set_dynamics_device): the leveller turned
    on where it was off, speed, amount, cap, gate and look-ahead changed elsewhere.  The running leveller state carries
    over the way the firmware's main loop keeps it (main.c:868-895): envelopes, gains, ring and index untouched, only
    the coefficients new."""
    q28 = flavour == "q28"
    n, fs, bd, frames, seed = LC.LEVEL_SETS["level24"]
    insts, P, bq, _ = LC.make_set(oracle, flavour, n, fs, bd, sum(frames), seed)
    P["leveller_enabled"][1::2] = 0
    oracle.set_libm_f64(1)
    r = Run(monkeypatch, oracle, flavour, insts, P, bq, 24 * 96)
    try:
        r.call([96] * 16)
        cfgs = np.zeros(n, L.DYNAMICS_CONFIG)
        cfgs["volume_8_8"] = -256                              # the host volume of the level set (-1 dB)
        cfgs["loudness_ref_spl"], cfgs["loudness_intensity_pct"] = 83.0, 100.0
        rng = np.random.default_rng(91)
        for i, it in enumerate(insts):
            c = it.case
            on_before = i % 2 == 0
            cfgs[i]["lev_enabled"] = 1
            cfgs[i]["lev_speed"] = c["speed"] if not on_before else (c["speed"] + 1 + int(rng.integers(4))) % 5
            cfgs[i]["lev_amount"] = c["amount"] if not on_before else float(rng.choice(LC.AMOUNTS))
            cfgs[i]["lev_max_gain_db"] = c["max_gain"] if not on_before else float(rng.choice(LC.MAX_GAINS))
            cfgs[i]["lev_gate_threshold_db"] = c["gate"] if not on_before else float(rng.choice(LC.GATES))
            cfgs[i]["lev_lookahead"] = c["lookahead"] if i % 4 != 0 else 1 - c["lookahead"]
        r.eng.set_dynamics_device(cfgs, fs)
        for i in range(n):
            apply_to_oracle(oracle, r.chains[i], cfgs[i], q28)
        r.state_check(LC.levs_record, "after set_dynamics_device (state untouched)")
        r.call([96] * 24)
    finally:
        r.close()
        oracle.set_libm_f64(0)
