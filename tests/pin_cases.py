"""Outputs of the oracle's per-function restatements on the inputs of tests/test_oracle_vs_ref.py, stored as
tests/golden/pins.npz so that the comparisons run where the reference sources are not present.

test_oracle_vs_ref.py checks these functions bit for bit against the reference compiled from its own sources; the
EQ coefficients and cascades, the whole chain, the bulk packet, preset slots and S/PDIF subframes already have
reference-made fixtures (tests/golden/make_golden*.py).  The vectors here were made with the restatement as of the
commit where it was last checked bit for bit against the compiled reference, so a change to the restatement that
moves it away from the reference shows up without the reference.

    python -m tests.pin_cases        # rewrites tests/golden/pins.npz
"""
import ctypes as C
import os

import numpy as np

from dspi_b200 import layouts as L
from dspi_b200 import workloads as W

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pins.npz")
FLAVOURS = ("f32s", "f32f", "q28")


def _xfeed_coeffs(oracle, q, preset, fs):
    cfg = (C.c_uint8 * 12)()
    c = np.frombuffer(cfg, np.uint8)
    c[0], c[1], c[2] = 1, 1, preset
    c[4:8] = np.frombuffer(np.float32(1234.0).tobytes(), np.uint8)
    c[8:12] = np.frombuffer(np.float32(7.0).tobytes(), np.uint8)
    st = np.zeros(1, L.XFEED_Q28 if q else L.XFEED_F32)
    (oracle.lib.orc_xfeed_coeffs_q28 if q else oracle.lib.orc_xfeed_coeffs_f32)(st.ctypes.data, C.addressof(cfg), fs)
    return st


def _lev_coeffs(oracle, level, speed, max_gain, gate, fs):
    cfg = np.zeros(24, np.uint8)
    cfg[0] = 1
    cfg[4:8] = np.frombuffer(np.float32(level).tobytes(), np.uint8)
    cfg[8] = speed
    cfg[12:16] = np.frombuffer(np.float32(max_gain).tobytes(), np.uint8)
    cfg[16] = 1
    cfg[20:24] = np.frombuffer(np.float32(gate).tobytes(), np.uint8)
    c = np.zeros(1, L.LEV_COEFFS)
    oracle.lib.orc_lev_coeffs_compute(c.ctypes.data, cfg.ctypes.data, fs)
    return c


def compute(oracle):
    """name -> array; every array is a pure function of the oracle and fixed seeds."""
    out = {}
    # fixed-point multiplies (test_q28_q15_multiplies)
    rng = np.random.default_rng(7)
    vals = np.concatenate([rng.integers(-2**31, 2**31, 4000, dtype=np.int64),
                           np.array([0, 1, -1, 2**31 - 1, -2**31, 1 << 28, -(1 << 28), 0xFFFF, 0x10000, -0x10000])])
    a, b = rng.permutation(vals)[:2000], rng.permutation(vals)[:2000]
    out["mul_q28"] = np.array([oracle.lib.orc_mul_q28(int(x), int(y)) for x, y in zip(a, b)], np.int32)
    out["mul_q15"] = np.array([oracle.lib.orc_mul_q15(int(x), int(y)) for x, y in zip(a, b)], np.int32)
    # crossfeed coefficients and filter (test_crossfeed)
    for fl in FLAVOURS:
        q = fl == "q28"
        for preset in range(4):
            st = _xfeed_coeffs(oracle, q, preset, 48000.0)
            out[f"xfeed_{fl}_{preset}_coeffs"] = st.view(np.uint8).copy()
            l, r = W.inputs_q28(2, 1000) if q else W.inputs_f32(2, 1000)
            l, r = l.copy(), r.copy()
            oracle.xfeed(fl, st, l, r)
            out[f"xfeed_{fl}_{preset}"] = np.stack([l, r])
            out[f"xfeed_{fl}_{preset}_state"] = st.view(np.uint8).copy()
    # leveller block loop, glibc float routines and x86 conversions as in test_leveller
    oracle.set_libm_f64(0)
    oracle.set_x86_cvt(1)
    try:
        coeffs = _lev_coeffs(oracle, 70.0, 2, 15.0, -80.0, 96000.0)
        for fl in FLAVOURS:
            q = fl == "q28"
            for lookahead in (0, 1):
                for count in (1, 48, 96):
                    st = np.zeros(1, L.LEV_STATE_Q28 if q else L.LEV_STATE_F32)
                    nblk = 20
                    if q:
                        l, r = W.inputs_q28(2, nblk * count)
                        l, r = l >> 3, r >> 4
                    else:
                        l, r = W.inputs_f32(2, nblk * count)
                        l, r = l * np.float32(0.1), r * np.float32(0.05)
                    l, r = np.ascontiguousarray(l), np.ascontiguousarray(r)
                    for k in range(nblk):
                        s = slice(k * count, (k + 1) * count)
                        ls, rs = l[s].copy(), r[s].copy()
                        oracle.leveller(fl, st, coeffs, lookahead, ls, rs)
                        l[s], r[s] = ls, rs
                    out[f"lev_{fl}_{lookahead}_{count}"] = np.stack([l, r])
                    out[f"lev_{fl}_{lookahead}_{count}_state"] = st.view(np.uint8).copy()
    finally:
        oracle.set_x86_cvt(0)
    # leveller coefficients and loudness tables (test_leveller_coeffs_and_loudness_tables)
    out["lev_coeffs"] = np.concatenate([_lev_coeffs(oracle, 55.0, s, 40.0, -100.0, 96000.0).view(np.uint8) for s in (0, 1, 2, 7)])
    for i, (spl, inten) in enumerate(((83.0, 100.0), (70.0, 50.0), (120.0, 150.0))):
        t = np.zeros((L.LOUD_STEPS, 2), L.LOUD_F32)
        oracle.lib.orc_loud_table_f32(t.ctypes.data, spl, inten, 96000.0)
        out[f"loud_f32_{i}"] = t.view(np.uint8).copy()
        t = np.zeros((L.LOUD_STEPS, 2), L.LOUD_Q28)
        oracle.lib.orc_loud_table_q28(t.ctypes.data, spl, inten, 96000.0)
        out[f"loud_q28_{i}"] = t.view(np.uint8).copy()
    # delay samples (test_delay_samples_and_volume_table)
    out["delay"] = np.array([[oracle.lib.orc_delay_samples(ms, fs, last, n) for n in (4096, 2048)]
                             for fs in (44100.0, 48000.0, 96000.0)
                             for ms in (0.0, 0.5, 10.0, 42.6, 85.3, 85.4, 1000.0, -3.0)
                             for last in (0, 1)], np.int32)
    return out


if __name__ == "__main__":
    from tests.orc import Oracle
    np.savez_compressed(PATH, **compute(Oracle()))
    print(PATH, os.path.getsize(PATH))
