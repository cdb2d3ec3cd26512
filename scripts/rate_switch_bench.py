"""Times a sample-rate switch of every instance of a chain engine, 8192 float and 8192 Q28 instances configured by
apply_bulk_device (packets from tests/bulk_cases.wire_packet seeds), switched 96 kHz <-> 48 kHz alternately:

  set_rate_device   dspi_chain(q)_set_rate_device; host clock around the call (it ends in a device synchronise), and CUDA
                    events on the engine stream around it
  workaround        collect_bulk_device + apply_bulk_device at the new rate (what a host could do before; it also converts
                    every gain again); host clock

Each is warmed up in both directions first; the report is the best of --reps alternating repetitions.  With --profile, a
separate run takes the rate kernel's own time per 1024-instance chunk from torch.profiler (CUDA activity).  Prints the card
and its power limit, read in the same run, and the bytes the switch moves, computed from the shapes.  Fails without a GPU."""
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

RATES = (48000.0, 96000.0)
CHUNK = 1024                                        # bulk::kChunk


def switch(eng, fs):
    import torch
    s = torch.cuda.ExternalStream(eng.stream)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rates = np.full(eng.n_instances, fs, np.float32)
    t0 = time.perf_counter()
    a.record(s)
    res = eng.set_rate_device(rates)
    b.record(s)
    b.synchronize()
    t1 = time.perf_counter()
    assert (res == L.BULK_CURRENT).all()
    return t1 - t0, a.elapsed_time(b) * 1e-3


def workaround(eng, fs):
    t0 = time.perf_counter()
    packets, host, marks = eng.collect_bulk_device()
    res = eng.apply_bulk_device(packets, fs, host=host)
    t1 = time.perf_counter()
    assert (marks == L.BULK_CURRENT).all() and not res.any()
    return t1 - t0


def profile(eng, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        for k in range(reps):
            switch(eng, RATES[k % 2])
    ev = [e for e in p.key_averages() if "rate_kernel" in e.key]
    assert ev, "no rate_kernel in the trace"
    calls = sum(e.count for e in ev)
    total_us = sum(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total for e in ev)
    return total_us / calls, calls


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="a separate run: the rate kernel's time per chunk from torch.profiler")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rate_switch_bench: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))
    N = a.instances
    for name, platform in (("f32f", L.PLATFORM_RP2350), ("q28", L.PLATFORM_RP2040)):
        q28 = platform == L.PLATFORM_RP2040
        roles = 7 if q28 else 11
        packets = np.concatenate([wire_packet(platform, 9000 + i) for i in range(N)])
        eng = api.ChainEngineQ28(N, 192) if q28 else api.ChainEngine(name, N, 192)
        assert not eng.apply_bulk_device(packets, RATES[1]).any()
        for fs in RATES:                                              # warm-up, both directions
            switch(eng, fs)
            workaround(eng, fs)
        out = {"case": f"{name} {N} instances, 96 <-> 48 kHz", "reps": a.reps}
        if a.profile:
            per_chunk_us, calls = profile(eng, a.reps)
            out["rate_kernel_us_per_chunk"] = round(per_chunk_us, 1)
            out["rate_kernel_launches"] = calls
        else:
            sw, wa = [], []
            for k in range(a.reps):                                   # alternating
                sw.append(switch(eng, RATES[k % 2]))
                wa.append(workaround(eng, RATES[(k + 1) % 2]))
            out["set_rate_device_ms"] = {"host_clock": round(min(s[0] for s in sw) * 1e3, 2),
                                         "engine_stream_events": round(min(s[1] for s in sw) * 1e3, 2)}
            out["collect_then_apply_ms"] = round(min(wa) * 1e3, 2)
        eng.close()
        bq = (L.BIQUAD_Q28 if q28 else L.BIQUAD_F32).itemsize
        out["mbytes"] = {"records_in": round(N * L.WIRE_BULK.itemsize / 1e6, 2),
                         "recipes_staged": round(N * roles * L.MAX_BANDS * 16 / 1e6, 2),      # written by the rate kernel, clamped in place, read back into the records
                         "mirror": round(N * roles * L.MAX_BANDS * bq / 1e6, 2)}             # unpacked, rewritten by the coefficient kernels, packed
        print(json.dumps(out))


if __name__ == "__main__":
    main()
