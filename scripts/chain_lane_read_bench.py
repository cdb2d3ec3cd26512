#!/usr/bin/env python
"""What lane read calls buy: G clock groups of n instances, each served on its own lane of one 8192-instance engine, with
one read per round on group 0, issued either as the engine-level getter (a barrier across every lane that also waits on
the host) or as the lane read on group 0's lane, into device memory.
    python scripts/chain_lane_read_bench.py [--ariths f32f,q28] [--groups 4,8] [--sizes 64,256] [--rounds 16] [--connections 8,32]

Float fused and Q28 chains, every instance configured from the firmware's default packet at 96 kHz, words and PDM out.
Even groups run 64 packets of 96 frames per call, odd groups the 10-packet 44.1 kHz cadence, so the groups' calls end out
of phase; every lane keeps two calls in flight (before a group's call is issued, its call of two rounds back is waited
for) and no round ends in a synchronisation.  Per round, group 0 first gets the read:
    none             no read
    getall-engine    dspi_chain(q)_collect_bulk_device of one instance of group 0 (a Console connecting: REQ_GET_ALL_PARAMS)
    getall-lane      dspi_chain(q)_lane_collect_bulk_device, the same on group 0's lane
    save-engine      dspi_chain(q)_collect_preset_device over group 0's window (a preset save)
    save-lane        the same on group 0's lane
    export-engine    dspi_chain(q)_export_instances of one instance of group 0 (a checkpoint, or a move to another GPU)
    export-lane      the same on group 0's lane
    response-engine  dspi_chain(q)_response_host over group 0's window at 256 frequencies (a Console's EQ curve)
    response-lane    dspi_chain(q)_lane_response_device, the same on group 0's lane
Reported per mode, after two warm-up rounds: host time inside the call (median and max, ms), p50 / p99 latency of the
untouched groups' calls from issue to completion (ms; an event recorded on an idle stream at issue and one on the lane
after the call, so both are on the GPU clock), and the mean round time (ms).  Each --connections value runs in a process of
its own with CUDA_DEVICE_MAX_CONNECTIONS set.  Every line carries the card name, power limit and max SM clock."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--instances", type=int, default=8192)
ap.add_argument("--ariths", default="f32f,q28")
ap.add_argument("--groups", default="4,8")
ap.add_argument("--sizes", default="64,256")
ap.add_argument("--rounds", type=int, default=16)
ap.add_argument("--connections", default="8,32")
ap.add_argument("--child", action="store_true")
a = ap.parse_args()
CADENCE = [44] * 9 + [45]
MODES = ["none", "getall-engine", "getall-lane", "save-engine", "save-lane", "export-engine", "export-lane", "response-engine", "response-lane"]
FS = 96000.0


def card(torch):
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        limit = q.stdout.strip() if q.returncode == 0 else "unknown"
    except (OSError, subprocess.TimeoutExpired):
        limit = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": limit}


def run_arith(arith, info):
    import numpy as np
    import torch
    from dspi_b200 import api, layouts as L

    N, F = a.instances, 64 * 96
    q28 = arith == "q28"
    eng = api.ChainEngineQ28(N, max_frames=F) if q28 else api.ChainEngine(arith, N, max_frames=F)
    plat = L.PLATFORM_RP2040 if q28 else L.PLATFORM_RP2350
    pk = api.bulk_params_collect(api.bulk_state_defaults(plat))
    assert (eng.apply_bulk_device(np.repeat(pk, N), FS) == 0).all()
    pcm = torch.randint(0, 256, (N, F * 6), dtype=torch.uint8, device="cuda")
    idle = torch.cuda.Stream()
    size, slot = eng.instance_image_size(), api.preset_slot_size(plat)
    freqs = np.geomspace(20.0, 20000.0, 256).astype(np.float32)
    try:
        for n in [int(x) for x in a.sizes.split(",")]:
            d_wire = torch.zeros((n, L.WIRE_BULK.itemsize), dtype=torch.uint8, device="cuda")
            d_host = torch.zeros((n, L.BULK_HOST.itemsize), dtype=torch.uint8, device="cuda")
            d_res = torch.zeros(n, dtype=torch.int32, device="cuda")
            d_img = torch.zeros((n, max(size, slot)), dtype=torch.uint8, device="cuda")
            d_resp = torch.zeros((n, eng._OUTS, 2, freqs.size), dtype=torch.complex64, device="cuda")
            for G in [int(x) for x in a.groups.split(",")]:
                if G * n > N:
                    continue
                tables = [np.array(CADENCE if g % 2 else [96] * 64, np.uint16) for g in range(G)]
                outs = [(torch.zeros((n, eng._PAIRS, int(t.sum()), 2), dtype=torch.int32, device="cuda"),
                         torch.zeros((n, int(t.sum()), 8), dtype=torch.int32, device="cuda")) for t in tables]
                torch.cuda.synchronize()
                lanes = [eng.lane_open(g * n, n) for g in range(G)]
                streams = [torch.cuda.ExternalStream(eng.lane_stream(ln)) for ln in lanes]
                try:
                    for mode in MODES:
                        host, lat, done = [], [], {}
                        t_start = None
                        for r in range(a.rounds + 2):
                            if r == 2:
                                torch.cuda.synchronize()
                                t_start = time.perf_counter()
                            i = r % n
                            t0 = time.perf_counter()
                            if mode == "getall-engine":
                                eng.collect_bulk_device(i, 1)
                            elif mode == "getall-lane":
                                eng.lane_collect_bulk_device(lanes[0], i, 1, d_wire.data_ptr(), d_host.data_ptr(), d_res.data_ptr())
                            elif mode == "save-engine":
                                eng.collect_preset_device(r % 10, 0, n)
                            elif mode == "save-lane":
                                eng.lane_collect_preset_device(lanes[0], r % 10, 0, d_img.data_ptr(), d_img.shape[1], n=n, results_ptr=d_res.data_ptr())
                            elif mode == "export-engine":
                                eng.export_instances(i, 1)
                            elif mode == "export-lane":
                                eng.lane_export_instances(lanes[0], i, 1, d_img.data_ptr(), d_img.shape[1])
                            elif mode == "response-engine":
                                eng.response(freqs, FS, 0, n)
                            elif mode == "response-lane":
                                eng.lane_response_device(lanes[0], freqs, FS, 0, n, d_resp.data_ptr())
                            if r >= 2 and mode != "none":
                                host.append((time.perf_counter() - t0) * 1e3)
                            for g in range(G):
                                if (g, r - 2) in done:
                                    done.pop((g, r - 2))[1].synchronize()
                                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                                ev0.record(idle)
                                sp, pd = outs[g]
                                eng.lane_process_packets_device(lanes[g], g * n, n, pcm.data_ptr() + g * n * pcm.shape[1], 24, tables[g],
                                                                sp.data_ptr(), pd.data_ptr())
                                ev1.record(streams[g])
                                done[(g, r)] = (ev0, ev1)
                                if r >= 2 and g > 0:
                                    lat.append((ev0, ev1))
                        for ln in lanes:
                            eng.lane_sync(ln)
                        round_ms = (time.perf_counter() - t_start) * 1e3 / a.rounds
                        ms = np.array([e0.elapsed_time(e1) for e0, e1 in lat])
                        out = {"arith": arith, "G": G, "n": n, "mode": mode, "round_ms": round(round_ms, 3),
                               "untouched_p50_ms": round(float(np.percentile(ms, 50)), 3), "untouched_p99_ms": round(float(np.percentile(ms, 99)), 3),
                               **info}
                        if host:
                            out["call_host_ms_median"], out["call_host_ms_max"] = round(float(np.median(host)), 4), round(float(np.max(host)), 4)
                        print(json.dumps(out), flush=True)
                finally:
                    for ln in lanes:
                        eng.lane_close(ln)
    finally:
        eng.close()


def run():
    import torch

    assert torch.cuda.is_available(), "chain_lane_read_bench needs a GPU"
    info = card(torch)
    info["max_connections"] = os.environ.get("CUDA_DEVICE_MAX_CONNECTIONS", "default (8)")
    for arith in a.ariths.split(","):
        run_arith(arith, info)


if __name__ == "__main__":
    if a.child:
        run()
    else:
        for k in a.connections.split(","):
            env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS=k)
            args = [sys.executable, os.path.abspath(__file__), "--child", "--instances", str(a.instances), "--ariths", a.ariths,
                    "--groups", a.groups, "--sizes", a.sizes, "--rounds", str(a.rounds)]
            subprocess.check_call(args, env=env)
