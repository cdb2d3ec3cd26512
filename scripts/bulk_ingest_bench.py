"""Times the two routes from WireBulkParams packets to a configured chain engine, side by side in one run, for 8192 float
and 8192 Q28 instances at 96 kHz (packets from tests/bulk_cases.wire_packet seeds):

  host route    dspi_bulk_params_apply + dspi_bulk_state_to_chain_* per instance in C through ctypes, then set_params +
                upload_biquads; host clock around calls that end in a device synchronise
  device route  dspi_chain(q)_apply_bulk_device; the same host clock, and CUDA events on the engine stream around the call
                (the span of its copies and kernels on the device)

Each route is warmed up once before it is timed.  Prints the card and its power limit, read in the same run, and the bytes
moved, computed from the shapes.  Fails without a GPU."""
import argparse
import ctypes as C
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


def host_route(eng, packets, platform, P, bq):
    h = api.lib()
    q28 = platform == L.PLATFORM_RP2040
    to_chain = h.dspi_bulk_state_to_chain_q28 if q28 else h.dspi_bulk_state_to_chain_f32
    st = np.zeros(1, L.BULK_STATE)
    sp, pk = st.ctypes.data_as(C.c_void_p), packets.ctypes.data
    t0 = time.perf_counter()
    for i in range(packets.shape[0]):
        h.dspi_bulk_state_defaults(sp, platform)
        h.dspi_bulk_params_apply(C.c_void_p(pk + i * L.WIRE_BULK.itemsize), sp, 0)
        to_chain(sp, C.c_float(FS), C.c_int16(0), 0, C.c_void_p(P.ctypes.data + i * P.dtype.itemsize),
                 C.c_void_p(bq.ctypes.data + i * bq[0].nbytes))
    t1 = time.perf_counter()
    eng.set_params(P)
    eng.upload_biquads(bq)
    t2 = time.perf_counter()
    return t1 - t0, t2 - t1


def device_route(eng, packets):
    import torch
    s = torch.cuda.ExternalStream(eng.stream)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record(s)
    res = eng.apply_bulk_device(packets, FS)
    b.record(s)
    b.synchronize()
    t1 = time.perf_counter()
    assert not res.any()
    return t1 - t0, a.elapsed_time(b) * 1e-3


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bulk_ingest_bench: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))
    N = a.instances
    for name, platform in (("f32f", L.PLATFORM_RP2350), ("q28", L.PLATFORM_RP2040)):
        q28 = platform == L.PLATFORM_RP2040
        roles, outs = (7, 5) if q28 else (11, 9)
        packets = np.concatenate([wire_packet(platform, 9000 + i) for i in range(N)])
        P = np.zeros(N, L.CHAIN_PARAMS_Q28 if q28 else L.CHAIN_PARAMS_F32)
        bq = np.zeros((N, roles, L.MAX_BANDS), L.BIQUAD_Q28 if q28 else L.BIQUAD_F32)
        eng = api.ChainEngineQ28(N, 192) if q28 else api.ChainEngine(name, N, 192)
        host_route(eng, packets, platform, P, bq)                     # warm-up of each route
        device_route(eng, packets)
        hs, dv = [], []
        for _ in range(a.reps):                                       # alternating
            hs.append(host_route(eng, packets, platform, P, bq))
            dv.append(device_route(eng, packets))
        eng.close()
        # SoA parameter rows written per instance: float engine 4 B x (2 preamp + 12 loudness + 7 crossfeed + 9 leveller +
        # 5 rows per output + 2 volume) + 1 B x (flags, loudness bypass, 2 master skip, 2 rows per output); Q28: 10 loudness words
        rows = 4 * (2 + (10 if q28 else 12) + 7 + 9 + 5 * outs + 2) + (4 + 2 * outs)
        mirror = roles * L.MAX_BANDS * (L.BIQUAD_Q28 if q28 else L.BIQUAD_F32).itemsize
        out = {
            "case": f"{name} {N} instances",
            "host_route_ms": {"per_instance_c": round(min(h[0] for h in hs) * 1e3, 2), "set_params_upload": round(min(h[1] for h in hs) * 1e3, 2),
                              "total": round(min(h[0] + h[1] for h in hs) * 1e3, 2)},
            "device_route_ms": {"host_clock": round(min(d[0] for d in dv) * 1e3, 2), "engine_stream_events": round(min(d[1] for d in dv) * 1e3, 2)},
            "mbytes": {"packets_in": round(N * L.WIRE_BULK.itemsize / 1e6, 2), "recipes": round(N * roles * L.MAX_BANDS * 16 / 1e6, 2),
                       "soa_rows_out": round(N * rows / 1e6, 2), "mirror_out": round(N * mirror / 1e6, 2)},
            "reps": a.reps,
        }
        print(json.dumps(out))


if __name__ == "__main__":
    main()
