"""Times the two directions of the bulk parameter interface on the device, side by side in one run, for 8192 float and 8192
Q28 instances at 96 kHz (packets from tests/bulk_cases.wire_packet seeds):

  apply    dspi_chain(q)_apply_bulk_device: wire bytes -> engine records and the configuration record of every instance
  collect  dspi_chain(q)_collect_bulk_device: configuration records -> wire bytes in host memory

Each call is timed with a host clock (it ends in a device synchronise) and with CUDA events on the engine stream (the span of
its copies and kernels on the device); best of alternating repetitions after one warm-up of each.  Prints the card and its
power limit, read in the same run, and the bytes each call moves, computed from the shapes.  Fails without a GPU."""
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


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bulk_collect_bench: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))
    N = a.instances
    for name, platform in (("f32f", L.PLATFORM_RP2350), ("q28", L.PLATFORM_RP2040)):
        q28 = platform == L.PLATFORM_RP2040
        packets = np.concatenate([wire_packet(platform, 9000 + i) for i in range(N)])
        eng = api.ChainEngineQ28(N, 192) if q28 else api.ChainEngine(name, N, 192)
        apply_call, collect_call = (lambda: eng.apply_bulk_device(packets, FS)), (lambda: eng.collect_bulk_device())
        timed(eng, apply_call)                                        # warm-up of each direction
        timed(eng, collect_call)
        ap_t, co_t = [], []
        for _ in range(a.reps):                                       # alternating
            t = timed(eng, apply_call)
            assert not t[2].any()
            ap_t.append(t[:2])
            t = timed(eng, collect_call)
            assert (t[2][2] == L.BULK_CURRENT).all() and (t[2][0]["header"]["format_version"] == 6).all()
            co_t.append(t[:2])
        eng.close()
        record = N * (L.WIRE_BULK.itemsize + L.BULK_HOST.itemsize + 1)
        out = {
            "case": f"{name} {N} instances",
            "apply_ms": {"host_clock": round(min(t[0] for t in ap_t) * 1e3, 2), "engine_stream_events": round(min(t[1] for t in ap_t) * 1e3, 2),
                         "host_clock_all": [round(t[0] * 1e3, 2) for t in ap_t]},
            "collect_ms": {"host_clock": round(min(t[0] for t in co_t) * 1e3, 2), "engine_stream_events": round(min(t[1] for t in co_t) * 1e3, 2),
                           "host_clock_all": [round(t[0] * 1e3, 2) for t in co_t]},
            # collect: record read, staging written, staging copied to the host (packet + host record + code per instance)
            "mbytes": {"record": round(record / 1e6, 2), "collect_device_traffic": round(2 * record / 1e6, 2),
                       "collect_to_host": round(N * (L.WIRE_BULK.itemsize + L.BULK_HOST.itemsize + 4) / 1e6, 2)},
            "reps": a.reps,
        }
        print(json.dumps(out))


if __name__ == "__main__":
    main()
