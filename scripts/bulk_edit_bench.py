"""Times sparse configuration edits of a chain engine, 8192 float and 8192 Q28 instances configured by apply_bulk_device at
96 kHz (packets from tests/bulk_cases.wire_packet seeds).  Cases, each an edit_bulk_device call:

  one        1 edit: one output gain of one instance
  band       one EQ band (16 bytes) on every instance
  mixed8     8 edits per instance: crosspoint gain, output gain, output mute, preamp, master volume, EQ band, crossfeed
             enable, host volume - interleaved across instances
  volume     a host-volume step on every instance

Each case is compared with the whole-instance route a host has otherwise (collect_bulk_device, the edits patched into the
packets in numpy, apply_bulk_device; the time of the two engine calls, the patch left out), and the band case also with
set_eq_params_device over every band of every instance.
Times are a host clock around a call that ends in a device synchronise; the report is the best of --reps alternating
repetitions after a warm-up.  A separate profiled run gives edit_kernel's device time per launch and its launches per call
(one per chunk of at most 1024 instances; torch.profiler, CUDA activity).  Prints the card and its power limit, read in
the same run.  Fails without a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dspi_b200 import api, layouts as L            # noqa: E402
from tests.bulk_cases import wire_packet            # noqa: E402

FS = 96000.0


def cases(N, outs, rng):
    inst = np.arange(N)
    one = L.bulk_edit(N // 3, ("outputs", 1, "gain_db"), np.float32(-4.0))
    band = np.repeat(L.bulk_edit(0, ("eq", 3, 5), (L.PEAKING, (0, 0, 0), 2500.0, 1.1, 4.5)), N)
    band["instance"] = inst
    per = [L.bulk_edit(0, ("crosspoints", 0, 1, "gain_db"), np.float32(-3.0)), L.bulk_edit(0, ("outputs", 2, "gain_db"), np.float32(-1.5)),
           L.bulk_edit(0, ("outputs", outs - 2, "mute"), 1), L.bulk_edit(0, ("preamp", "preamp_db", 1), np.float32(-2.0)),
           L.bulk_edit(0, ("master_volume", "master_volume_db"), np.float32(-9.0)),
           L.bulk_edit(0, ("eq", 2, 7), (L.HIGHSHELF, (0, 0, 0), 6000.0, 0.7, -3.0)), L.bulk_edit(0, ("crossfeed", "enabled"), 1),
           L.bulk_edit(0, ("host", "volume_8_8"), -15 * 256)]
    mixed = np.concatenate([np.repeat(e, N) for e in per])
    mixed["instance"] = np.tile(inst, len(per))
    mixed = mixed[rng.permutation(mixed.shape[0])]
    volume = np.repeat(L.bulk_edit(0, ("host", "volume_8_8"), -20 * 256), N)
    volume["instance"] = inst
    return {"one": one, "band": band, "mixed8": mixed, "volume": volume}


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return time.perf_counter() - t0, r


def edit_call(eng, edits):
    res = eng.edit_bulk_device(edits, FS)
    assert (res == L.BULK_CURRENT).all()


def route(eng, edits):
    """collect, the edits written over packets and host records in list order, apply; returns the seconds of the two
    engine calls (the numpy patch between them is left out, so the route is not charged for Python)"""
    t0 = time.perf_counter()
    P, H, marks = eng.collect_bulk_device()
    t1 = time.perf_counter()
    n = P.shape[0]
    buf = np.concatenate([P.view(np.uint8).reshape(n, 2896), H.view(np.uint8).reshape(n, 4)], axis=1)
    for e in edits:
        o, k = int(e["offset"]), int(e["length"])
        buf[int(e["instance"]), o:o + k] = e["bytes"][:k]
    P2 = np.ascontiguousarray(buf[:, :2896]).view(L.WIRE_BULK).reshape(n)
    H2 = np.ascontiguousarray(buf[:, 2896:]).view(L.BULK_HOST).reshape(n)
    t2 = time.perf_counter()
    res = eng.apply_bulk_device(P2, FS, host=H2)
    t3 = time.perf_counter()
    assert (marks == L.BULK_CURRENT).all() and not res.any()
    return (t1 - t0) + (t3 - t2)


def eq_params_call(eng, recipes):
    eng.set_eq_params_device(recipes, FS)


def all_recipes(eng, roles):
    """every band of every instance as set_eq_params_device takes them, from the records"""
    P = eng.collect_bulk_device()[0]
    r = np.zeros((P.shape[0], roles, L.MAX_BANDS), L.EQ_PARAM)
    eq = P["eq"][:, :roles]
    r["channel"] = np.arange(roles)[None, :, None]
    r["band"] = np.arange(L.MAX_BANDS)[None, None, :]
    for f, g in (("type", "type"), ("freq", "freq"), ("Q", "q"), ("gain_db", "gain_db")):
        r[f] = eq[g]
    return r


def profile(eng, edits, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(reps):
            edit_call(eng, edits)
    ev = [e for e in p.key_averages() if "edit_kernel" in e.key]
    assert ev, "no edit_kernel in the trace"
    calls = sum(e.count for e in ev)
    total_us = sum(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total for e in ev)
    return total_us / calls, calls / reps


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="a separate run: edit_kernel's device time per launch")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bulk_edit_bench: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))
    N = a.instances
    for name, platform in (("f32f", L.PLATFORM_RP2350), ("q28", L.PLATFORM_RP2040)):
        q28 = platform == L.PLATFORM_RP2040
        roles, outs = (7, 5) if q28 else (11, 9)
        packets = np.concatenate([wire_packet(platform, 12000 + i, version=6) for i in range(N)])
        eng = api.ChainEngineQ28(N, 192) if q28 else api.ChainEngine(name, N, 192)
        assert not eng.apply_bulk_device(packets, FS).any()
        cs = cases(N, outs, np.random.default_rng(1))
        recipes = all_recipes(eng, roles)
        for edits in cs.values():                                    # warm-up
            edit_call(eng, edits)
            route(eng, edits)
        eq_params_call(eng, recipes)
        for case, edits in cs.items():
            out = {"engine": f"{name} {N} instances at 96 kHz", "case": case, "edits": int(edits.shape[0]), "reps": a.reps}
            if a.profile:
                kern_us, launches = profile(eng, edits, a.reps)
                out["edit_kernel_us_per_launch"] = round(kern_us, 1)
                out["edit_kernel_launches_per_call"] = launches
            else:
                ed, ro, eqp = [], [], []
                for _ in range(a.reps):                              # alternating
                    ed.append(timed(lambda: edit_call(eng, edits))[0])
                    ro.append(route(eng, edits))
                    if case == "band":
                        eqp.append(timed(lambda: eq_params_call(eng, recipes))[0])
                out["edit_bulk_device_ms"] = round(min(ed) * 1e3, 3)
                out["collect_and_apply_ms"] = round(min(ro) * 1e3, 3)
                if eqp:
                    out["set_eq_params_device_ms"] = round(min(eqp) * 1e3, 3)
            print(json.dumps(out))
        eng.close()


if __name__ == "__main__":
    main()
