#!/usr/bin/env python
"""What lane move calls buy: G clock groups of n instances, each served on its own lane of one 8192-instance engine, with
one move per round on group 0 or from group 0 into group 1, issued either as engine-level calls (barriers across every
lane that also wait on the host) or as lane calls.
    python scripts/chain_lane_move_bench.py [--ariths f32f,q28] [--groups 4,8] [--sizes 64,256] [--rounds 16] [--connections 8,32]

Float fused and Q28 chains, every instance configured from the firmware's default packet at 96 kHz, words and PDM out.
Even groups run 64 packets of 96 frames per call, odd groups the 10-packet 44.1 kHz cadence, so the groups' calls end out
of phase; every lane keeps two calls in flight (before a group's call is issued, its call of two rounds back is waited
for) and no round ends in a synchronisation.  Per round, before the process calls:
    none            no move
    rate-engine     dspi_chain(q)_set_rate_device of one device of group 0 (48 and 96 kHz in turn), then
                    dspi_chain(q)_copy_instances of it into group 1 (a device changing rate moves to another group)
    rate-lane       dspi_chain(q)_lane_set_rate_device on group 0's lane, then _lane_copy_instances from group 0's lane
                    to group 1's
    repack-engine   dspi_chain(q)_copy_instances of min(64, n / 2) devices within group 0 (a group repacking its slots)
    repack-lane     the same with _lane_copy_instances on group 0's lane
    connect-engine  dspi_chain(q)_import_instances of one image into group 0 (a device connecting from a checkpoint)
    connect-lane    dspi_chain(q)_lane_import_instances, the same on group 0's lane
    restore-engine  dspi_chain(q)_import_instances of group 0's whole window (a group restored from a checkpoint)
    restore-lane    the same on group 0's lane
Reported per mode, after --warmup rounds (default 8, so that every buffer of a lane's ring of 8 pinned host buffers has
grown to the mode's upload; a growth frees pinned memory, which waits for the device): host time inside the move (median
and max, ms; both calls of a rate move), p50 / p99 latency of the untouched groups' calls from issue to completion (ms;
an event recorded on an idle stream at issue and one on the lane after the call, so both are on the GPU clock; groups 0
and 1 are the touched ones), and the mean round time (ms).  Each --connections value runs in a process of its own with
CUDA_DEVICE_MAX_CONNECTIONS set.  Every line carries the card name, power limit and max SM clock."""
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
ap.add_argument("--warmup", type=int, default=8)
ap.add_argument("--connections", default="8,32")
ap.add_argument("--child", action="store_true")
a = ap.parse_args()
CADENCE = [44] * 9 + [45]
MODES = ["none", "rate-engine", "rate-lane", "repack-engine", "repack-lane", "connect-engine", "connect-lane", "restore-engine", "restore-lane"]
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
    d_res = torch.zeros(N, dtype=torch.int32, device="cuda")
    try:
        for n in [int(x) for x in a.sizes.split(",")]:
            images = eng.export_instances(0, n)
            k = min(64, n // 2)
            for G in [int(x) for x in a.groups.split(",")]:
                if G * n > N or G < 2:
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
                        for r in range(a.rounds + a.warmup):
                            if r == a.warmup:
                                torch.cuda.synchronize()
                                t_start = time.perf_counter()
                            s, d = r % n, n + r % n
                            rate = np.array([(48000.0, FS)[r % 2]], np.float32)
                            t0 = time.perf_counter()
                            if mode == "rate-engine":
                                eng.set_rate_device(rate, inst0=s)
                                eng.copy_instances([s], [d])
                            elif mode == "rate-lane":
                                eng.lane_set_rate_device(lanes[0], rate, s, results_ptr=d_res.data_ptr())
                                eng.lane_copy_instances(lanes[0], lanes[1], [s], [d])
                            elif mode == "repack-engine":
                                eng.copy_instances(np.arange(k), np.arange(k, 2 * k))
                            elif mode == "repack-lane":
                                eng.lane_copy_instances(lanes[0], lanes[0], np.arange(k), np.arange(k, 2 * k))
                            elif mode == "connect-engine":
                                eng.import_instances(images[s:s + 1], inst0=s)
                            elif mode == "connect-lane":
                                eng.lane_import_instances(lanes[0], images[s:s + 1], s)
                            elif mode == "restore-engine":
                                eng.import_instances(images, inst0=0)
                            elif mode == "restore-lane":
                                eng.lane_import_instances(lanes[0], images, 0)
                            if r >= a.warmup and mode != "none":
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
                                if r >= a.warmup and g > 1:
                                    lat.append((ev0, ev1))
                        for ln in lanes:
                            eng.lane_sync(ln)
                        round_ms = (time.perf_counter() - t_start) * 1e3 / a.rounds
                        ms = np.array([e0.elapsed_time(e1) for e0, e1 in lat])
                        out = {"arith": arith, "G": G, "n": n, "mode": mode, "moved": 1 if mode[:3] in ("rat", "con") else k if mode[:3] == "rep" else n,
                               "round_ms": round(round_ms, 3),
                               "untouched_p50_ms": round(float(np.percentile(ms, 50)), 3), "untouched_p99_ms": round(float(np.percentile(ms, 99)), 3),
                               **info}
                        if host:
                            out["call_host_ms_median"], out["call_host_ms_max"] = round(float(np.median(host)), 4), round(float(np.max(host)), 4)
                        print(json.dumps(out), flush=True)
                    eng.import_instances(images, inst0=0)
                finally:
                    for ln in lanes:
                        eng.lane_close(ln)
    finally:
        eng.close()


def run():
    import torch

    assert torch.cuda.is_available(), "chain_lane_move_bench needs a GPU"
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
                    "--groups", a.groups, "--sizes", a.sizes, "--rounds", str(a.rounds), "--warmup", str(a.warmup)]
            subprocess.check_call(args, env=env)
