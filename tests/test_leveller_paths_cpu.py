"""The leveller's level-dependent paths on the CPU: a census that proves the signals of tests/leveller_cases.py reach every
block decision of the leveller (gate, boost, knee, compression, max-gain clamp), its peak limiter and the Q28 gain
saturation in every flavour; the oracle's leveller against the compiled leveller.c on those signals; and the libm-policy
deviation (DESIGN.md §6) measured on them.

The GPU tests (test_leveller_paths_gpu.py) run the same sets, so a signal edited until it no longer reaches a branch
fails here first."""
import numpy as np
import pytest

from tests import leveller_cases as LC
from tests.orc import orc_chain_run, orc_chain_run_q28

FLAVOURS = ["f32f", "f32s", "q28"]
MIN_BLOCKS = 30                  # "a few dozen" blocks of every outcome, per flavour


@pytest.mark.parametrize("flavour", FLAVOURS)
def test_census_reaches_every_leveller_path(oracle, flavour):
    oracle.set_libm_f64(1)
    try:
        total = {}
        rows = []
        for name, (n, fs, bd, frames, seed) in LC.LEVEL_SETS.items():
            insts, P, bq, _ = LC.make_set(oracle, flavour, n, fs, bd, sum(frames), seed)
            c = LC.census(oracle, flavour, insts, P, bq, frames)
            rows.append((name, c))
            for k, v in c.items():
                total[k] = total.get(k, 0) + v
    finally:
        oracle.set_libm_f64(0)
    keys = LC.OUTCOMES + ("saturated", "nan", "blocks")
    print(f"\nleveller census, {flavour} (blocks per outcome; limiter = blocks where it acts on >= 1 sample)")
    print("set      " + " ".join(f"{k:>11}" for k in keys))
    for name, c in rows + [("total", total)]:
        print(f"{name:8} " + " ".join(f"{c[k]:>11}" for k in keys))
    for k in LC.OUTCOMES:
        assert total[k] >= MIN_BLOCKS, f"{flavour}: only {total[k]} blocks reach '{k}'"
    if flavour == "q28":
        assert total["saturated"] >= MIN_BLOCKS, "the Q28 gain cast never saturates (gain > 8 needs > 18.06 dB)"
        assert total["nan"] >= MIN_BLOCKS, "no Q28 envelope below zero (tiny negative samples)"
    else:
        assert total["saturated"] == 0 and total["nan"] == 0


def test_settled_state_round_trips_through_the_state_blob_layout():
    """blob_leveller() reads the sections where instance_arrays() puts them: a synthetic blob with every row numbered."""
    for q28 in (False, True):
        N = 37
        Np = 64
        hdr = 32 if q28 else 40
        words = 15 * Np + 5 * Np + Np + 2 * LC.LA * Np
        blob = np.zeros(hdr + 4 * words, np.uint8)
        h = blob[:hdr].view(np.uint32)
        h[0], h[1], h[3] = 0x53505344, 1 if q28 else 2, N
        w = blob[hdr:].view(np.uint32)
        w[:] = np.arange(words, dtype=np.uint32)
        v = {k: a.view(np.uint32) for k, a in LC.blob_leveller(blob, q28, N).items()}
        base = 15 * Np
        assert v["env_sq_l"][3] == base + 3 and v["env_sq_r"][5] == base + Np + 5
        if q28:
            assert v["gain_q28"][0] == base + 2 * Np and v["gain_prev_q28"][1] == base + 3 * Np + 1
            assert v["gain_smooth_db"][2] == base + 4 * Np + 2
        else:
            assert v["gain_smooth_db"][2] == base + 2 * Np + 2
            assert v["gain_linear"][0] == base + 3 * Np and v["gain_prev_linear"][1] == base + 4 * Np + 1
        assert v["la_write_idx"][36] == base + 5 * Np + 36
        assert v["lookahead_buf"][7, 1, 9] == base + 6 * Np + (LC.LA + 9) * Np + 7
        v["la_write_idx"][4] = 0xABCDEF
        assert w[base + 5 * Np + 4] == 0xABCDEF                     # the views write into the blob


@pytest.mark.parametrize("count", [1, 47, 96])
@pytest.mark.parametrize("flavour", FLAVOURS)
def test_oracle_leveller_equals_compiled_reference_on_paths(oracle, refs, flavour, count):
    """leveller.c compiled unmodified (oracle/_ref) against the oracle in its glibc flavour and x86 conversions, on every
    instance of the 24-bit level set from its settled state: outputs and state bit-exact, block after block."""
    q28 = flavour == "q28"
    n, fs, bd, _, seed = LC.LEVEL_SETS["level24"]
    nblk = 600 // count if count == 1 else 30
    insts = LC.instances(n, fs, nblk * count, bd, seed)
    oracle.set_libm_f64(0)
    oracle.set_x86_cvt(1)          # the x86 reference objects use CVTTSS2SI for the gain-cap and max_g casts
    try:
        for i, it in enumerate(insts):
            coeffs = np.array([it.lc], it.lc.dtype)
            st_orc, st_ref = it.settled(q28), it.settled(q28)
            x = LC.leveller_input(it.body, bd, q28)
            l1, r1 = np.ascontiguousarray(x[:, 0]), np.ascontiguousarray(x[:, 1])
            l2, r2 = l1.copy(), r1.copy()
            la = it.case["lookahead"]
            for k in range(nblk):
                s = slice(k * count, (k + 1) * count)
                a, b, c, d = l1[s].copy(), r1[s].copy(), l2[s].copy(), r2[s].copy()
                oracle.leveller(flavour, st_orc, coeffs, la, a, b)
                refs[flavour].leveller(st_ref, coeffs, la, c, d)
                l1[s], r1[s], l2[s], r2[s] = a, b, c, d
                assert st_orc.tobytes() == st_ref.tobytes(), f"instance {i} {it.case}: state after block {k}"
            assert l1.tobytes() == l2.tobytes() and r1.tobytes() == r2.tobytes(), f"instance {i} {it.case}: output"
    finally:
        oracle.set_x86_cvt(0)
        oracle.set_libm_f64(0)


def _words(oracle, flavour, insts, P, bq, pcm, bd, frames, mode):
    oracle.set_libm_f64(mode)
    try:
        q28 = flavour == "q28"
        out = []
        for i, it in enumerate(insts):
            ch = LC.oracle_chain(oracle, q28, P[i], bq[i], it)
            if q28:
                out.append(orc_chain_run_q28(oracle, ch, pcm[i], bd, len(frames), frames[0])[0])
            else:
                out.append(orc_chain_run(oracle, flavour, ch, pcm[i], bd, len(frames), frames[0])[0])
        return np.stack(out)
    finally:
        oracle.set_libm_f64(0)


# Measured on the CPU (x86-64, glibc) against the policy flavour, per group of sets: "level" = both level sets,
# "stages" = the 24-bit set with loudness, crossfeed and master EQ on.  Max |difference| of a 24-bit S/PDIF word in LSB,
# and the share of words that differ:
#   f32f  level   1 LSB, 0.033 %     stages  1 LSB, 0.008 %
#   f32s  level   9 LSB, 0.12 %      stages  1 LSB, 0.008 %
#   q28   level   1 LSB, 0.004 %     stages  175 LSB, 0.28 %
# f32s: where the block gain differs by one ulp, the per-sample ramp (gain += step, rounded at every sample) carries the
# difference on through the packet; the largest, 9 LSB (7 with every output EQ flat), is on a noise instance whose gain
# ramps up through unity.  q28 "stages": the
# truncating Q28 output EQs turn a 1-LSB input change into their own round-off noise (DESIGN.md §6).  Bounds: about twice
# the measurement, the Q28 noise-floor bound of §6 (-72 dBFS) behind the Q28 EQs.
BOUNDS = {("f32f", "level"): (2, 2e-3), ("f32f", "stages"): (2, 5e-4),
          ("f32s", "level"): (16, 4e-3), ("f32s", "stages"): (2, 5e-4),
          ("q28", "level"): (2, 5e-4), ("q28", "stages"): (int((1 << 23) * 10 ** (-72 / 20)), 1e-2)}


@pytest.mark.parametrize("flavour", FLAVOURS)
def test_libm_policy_deviation_on_paths(oracle, flavour):
    """The GPU's libm policy (double, rounded once) against the glibc flavour that oracle/_ref pins, on the path signals:
    gated, boosted, clamped, limited, saturated and NaN blocks included."""
    groups = {"level": [(k, False) for k in LC.LEVEL_SETS], "stages": [("level24", True)]}
    for group, sets in groups.items():
        worst, diff, words = 0, 0, 0
        for name, stages in sets:
            n, fs, bd, frames, seed = LC.LEVEL_SETS[name]
            insts, P, bq, pcm = LC.make_set(oracle, flavour, n, fs, bd, sum(frames), seed, stages=stages)
            a = _words(oracle, flavour, insts, P, bq, pcm, bd, frames, 0)
            b = _words(oracle, flavour, insts, P, bq, pcm, bd, frames, 1)
            d = np.abs(a.astype(np.int64) - b)
            worst, diff, words = max(worst, int(d.max())), diff + int((d > 0).sum()), words + d.size
        frac = diff / words
        print(f"\n{flavour} {group}: max deviation {worst} LSB, {diff} of {words} words differ ({100 * frac:.4f} %)")
        want_max, want_frac = BOUNDS[(flavour, group)]
        assert worst <= want_max and frac < want_frac, f"{flavour} {group}: {worst} LSB, {100 * frac:.4f} % of the words"
