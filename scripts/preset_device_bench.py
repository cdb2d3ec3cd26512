"""Times preset slot images on the device against the host routes, for 8192 float and 8192 Q28 instances at 96 kHz (images
from tests/bulk_cases.wire_packet seeds, written by dspi_preset_slot_collect):

  apply        dspi_chain(q)_apply_preset_device: slot images -> engine records
  host_bulk    per instance dspi_preset_slot_apply + dspi_bulk_params_collect on the host, then one apply_bulk_device(exact_db = 1)
  host_params  per instance dspi_preset_slot_apply + dspi_bulk_state_to_chain_* on the host, then set_params + upload_biquads
  collect      dspi_chain(q)_collect_preset_device: configuration records -> slot images in host memory
  host_collect collect_bulk_device, then per instance dspi_bulk_params_apply + dspi_preset_slot_collect on the host

The host routes loop over the C functions from Python, as a host program without its own C loop would.  Every call is timed
with a host clock around work that ends in a device synchronise, the device calls also with CUDA events on the engine stream;
best of alternating repetitions after one warm-up of each.  Then, in a profiled call of its own, the kernel times of one
apply: the decode kernel per 1024-instance chunk against the ingest kernel it feeds.  Prints the card and its power limit,
read in the same run.  Fails without a GPU."""
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


def timed(eng, call):
    import torch
    s = torch.cuda.ExternalStream(eng.stream)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record(s)
    out = call()
    b.record(s)
    b.synchronize()
    t1 = time.perf_counter()
    return t1 - t0, a.elapsed_time(b) * 1e-3, out


def kernel_times(eng, call):
    """mean device time per launch of the decode and ingest kernels over one call, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for key in ("preset_decode_kernel", "bulk_ingest_kernel"):
            if key in ev.key:
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                out[key] = {"launches": ev.count, "us_per_launch": round(t / max(ev.count, 1), 1)}
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("preset_device_bench: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))
    N = a.instances
    for name, platform in (("f32f", L.PLATFORM_RP2350), ("q28", L.PLATFORM_RP2040)):
        q28 = platform == L.PLATFORM_RP2040
        slots = (np.arange(N) % 10).astype(np.uint8)
        images = []
        for i in range(N):
            st = api.bulk_state_defaults(platform)
            assert api.bulk_params_apply(wire_packet(platform, 9000 + i), st, True) == 0
            images.append(api.preset_slot_collect(st, int(slots[i])))
        images = np.stack(images)
        eng = api.ChainEngineQ28(N, 192) if q28 else api.ChainEngine(name, N, 192)

        def apply_call():
            return eng.apply_preset_device(images, FS, slots=slots, master_volume_mode=1)

        def host_bulk():
            packets = []
            for i in range(N):
                st = api.bulk_state_defaults(platform)
                assert api.preset_slot_apply(images[i], int(slots[i]), st, 1, 0.0) == 0
                packets.append(api.bulk_params_collect(st))
            return eng.apply_bulk_device(np.concatenate(packets), FS, exact_db=True)

        def host_params():
            Ps = np.zeros(N, L.CHAIN_PARAMS_Q28 if q28 else L.CHAIN_PARAMS_F32)
            bqs = np.zeros((N, 7 if q28 else 11, L.MAX_BANDS), L.BIQUAD_Q28 if q28 else L.BIQUAD_F32)
            for i in range(N):
                st = api.bulk_state_defaults(platform)
                assert api.preset_slot_apply(images[i], int(slots[i]), st, 1, 0.0) == 0
                P, _ = api.bulk_state_to_chain(st, FS, biquads=bqs[i:i + 1])
                Ps[i] = P[0]
            eng.set_params(Ps)
            eng.upload_biquads(bqs)

        def collect_call():
            return eng.collect_preset_device(slots)

        def host_collect():
            packets = eng.collect_bulk_device()[0]
            out = np.zeros_like(images)
            for i in range(N):
                st = api.bulk_state_defaults(platform)
                assert api.bulk_params_apply(packets[i:i + 1], st, True) == 0
                out[i] = api.preset_slot_collect(st, int(slots[i]))
            return out

        calls = {"apply": apply_call, "host_bulk": host_bulk, "host_params": host_params}
        times = {k: [] for k in (*calls, "collect", "host_collect")}
        for k, c in calls.items():                                    # warm-up of each
            timed(eng, c)
        apply_call()
        timed(eng, collect_call)
        timed(eng, host_collect)
        for _ in range(a.reps):                                       # alternating
            for k, c in calls.items():
                times[k].append(timed(eng, c)[:2])
            apply_call()                                              # the collect directions read what the device apply wrote
            t = timed(eng, collect_call)
            assert (t[2][1] == L.BULK_CURRENT).all()
            times["collect"].append(t[:2])
            t = timed(eng, host_collect)
            assert np.array_equal(t[2], eng.collect_preset_device(slots)[0]), "device and host collect disagree"
            times["host_collect"].append(t[:2])
        kt = kernel_times(eng, apply_call)
        eng.close()
        out = {"case": f"{name} {N} instances", "reps": a.reps, "kernels_in_one_apply": kt}
        for k, ts in times.items():
            out[k + "_ms"] = {"host_clock": round(min(t[0] for t in ts) * 1e3, 2), "engine_stream_events": round(min(t[1] for t in ts) * 1e3, 2),
                              "host_clock_all": [round(t[0] * 1e3, 2) for t in ts]}
        print(json.dumps(out))


if __name__ == "__main__":
    main()
