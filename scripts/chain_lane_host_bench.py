#!/usr/bin/env python
"""What lane host calls buy: G clock groups of n instances, each served on its own lane of one engine, from page-locked host
memory (PCM in, S/PDIF and PDM out), against the other ways a host-resident farm can run them.
    python scripts/chain_lane_host_bench.py [--ariths f32f,q28] [--groups 2,4,8] [--sizes 64,256,1024] [--forms words,subframes]
                                            [--rounds 5] [--warmup 2] [--connections 8,32]

Every instance is configured from the firmware's default packet at 96 kHz; every call is 64 packets of 96 frames, 24-bit
PCM in, S/PDIF words or subframes and PDM out.  A round issues one call per group and ends when every group's call has
finished; the time per round is the mean over --rounds rounds after --warmup.  Variants:
    a  lane host calls: dspi_chain(q)_lane_process_packets_host / _subframes_host
    b  lane device calls on device-resident buffers (the device time, no copies)
    c  lane device calls with the caller's whole-buffer cudaMemcpyAsync of the PCM before and of the outputs after, on the
       lane stream
    d  the engine-level dspi_chain(q)_process_packets_range_host / _subframes_range_host, one group after another
Also reported: the host time inside a call (median, ms) of a and d; the pinned host-to-device and device-to-host bandwidth
measured in the same run (1 GiB copies) and the link time of a round from them (the larger of bytes in / H2D and bytes out
/ D2H); the card name, power limit and max SM clock.  Each --connections value runs in a process of its own with
CUDA_DEVICE_MAX_CONNECTIONS set."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--ariths", default="f32f,q28")
ap.add_argument("--groups", default="2,4,8")
ap.add_argument("--sizes", default="64,256,1024")
ap.add_argument("--forms", default="words,subframes")
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--connections", default="8,32")
ap.add_argument("--child", action="store_true")
a = ap.parse_args()
FS = 96000.0
NPK, FPP = 64, 96


def card(torch):
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        limit = q.stdout.strip() if q.returncode == 0 else "unknown"
    except (OSError, subprocess.TimeoutExpired):
        limit = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": limit}


def link(torch):
    """pinned host-to-device and device-to-host GB/s over 1 GiB copies"""
    nb = 1 << 30
    h = torch.empty(nb, dtype=torch.uint8).pin_memory()
    d = torch.empty(nb, dtype=torch.uint8, device="cuda")
    out = {}
    for what, dst, src in (("h2d", d, h), ("d2h", h, d)):
        dst.copy_(src, non_blocking=True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            dst.copy_(src, non_blocking=True)
        e1.record()
        e1.synchronize()
        out[what] = 3 * nb / (e0.elapsed_time(e1) * 1e-3) / 1e9
    del h, d
    return out


def run_arith(arith, info, bw):
    import numpy as np
    import torch
    from dspi_b200 import api, layouts as L

    # the caller's whole-buffer copies of variant c, on the lane stream (through the driver, so that torch keeps no record
    # of a lane stream that closes before the buffers are freed)
    drv = C.CDLL("libcuda.so.1")
    drv.cuMemcpyHtoDAsync_v2.argtypes = [C.c_uint64, C.c_void_p, C.c_size_t, C.c_void_p]
    drv.cuMemcpyDtoHAsync_v2.argtypes = [C.c_void_p, C.c_uint64, C.c_size_t, C.c_void_p]

    def copy(fn, dst, src, s):
        assert fn(dst.data_ptr(), src.data_ptr(), src.numel() * src.element_size(), s) == 0

    sizes, groups = [int(x) for x in a.sizes.split(",")], [int(x) for x in a.groups.split(",")]
    N, F = max(g * n for g in groups for n in sizes), NPK * FPP
    q28 = arith == "q28"
    eng = api.ChainEngineQ28(N, max_frames=F) if q28 else api.ChainEngine(arith, N, max_frames=F)
    plat = L.PLATFORM_RP2040 if q28 else L.PLATFORM_RP2350
    pk = api.bulk_params_collect(api.bulk_state_defaults(plat))
    assert (eng.apply_bulk_device(np.repeat(pk, N), FS) == 0).all()
    P = eng._PAIRS
    table = np.full(NPK, FPP, np.uint16)
    pcm_h = torch.randint(0, 256, (N, F * 6), dtype=torch.uint8).pin_memory()
    pcm_d = pcm_h.cuda()
    sp_h = torch.zeros(N * P * F * 4, dtype=torch.int32).pin_memory()       # room for subframes
    pd_h = torch.zeros(N * F * 8, dtype=torch.int32).pin_memory()
    sp_d, pd_d = torch.zeros_like(sp_h, device="cuda"), torch.zeros_like(pd_h, device="cuda")
    try:
        for form in a.forms.split(","):
            sub = form == "subframes"
            w = 4 if sub else 2
            name = "subframes" if sub else "packets"
            host_fn = eng._fn("process_%s_range_host" % name)
            for n in sizes:
                for G in groups:
                    if G * n > N:
                        continue
                    rows = lambda buf, g, per: buf[g * n * per:(g + 1) * n * per]   # noqa: E731
                    pcm_hg = [pcm_h[g * n:(g + 1) * n] for g in range(G)]
                    pcm_dg = [pcm_d[g * n:(g + 1) * n] for g in range(G)]
                    sp_hg = [rows(sp_h, g, P * F * w) for g in range(G)]
                    sp_dg = [rows(sp_d, g, P * F * w) for g in range(G)]
                    pd_hg = [rows(pd_h, g, F * 8) for g in range(G)]
                    pd_dg = [rows(pd_d, g, F * 8) for g in range(G)]
                    torch.cuda.synchronize()
                    lanes = [eng.lane_open(g * n, n) for g in range(G)]
                    out = {"arith": arith, "form": form + "+pdm", "G": G, "n": n, "frames": F}
                    try:
                        for v in "abcd":
                            host = []
                            t_start = None
                            for r in range(a.rounds + a.warmup):
                                if r == a.warmup:
                                    torch.cuda.synchronize()
                                    t_start = time.perf_counter()
                                for g in range(G):
                                    t0 = time.perf_counter()
                                    if v == "a":
                                        eng.lane_process_packets_host(lanes[g], g * n, pcm_hg[g], 24, table, sp_hg[g], pd_hg[g], subframes=sub)
                                    elif v == "d":
                                        assert host_fn(eng._h, g * n, n, C.c_void_p(pcm_hg[g].data_ptr()), 24, NPK, table.ctypes.data,
                                                       C.c_void_p(sp_hg[g].data_ptr()), C.c_void_p(pd_hg[g].data_ptr()), None) == 0
                                    else:
                                        s = C.c_void_p(eng.lane_stream(lanes[g]))
                                        if v == "c":
                                            copy(drv.cuMemcpyHtoDAsync_v2, pcm_dg[g], pcm_hg[g], s)
                                        getattr(eng, "lane_process_%s_device" % name)(lanes[g], g * n, n, pcm_dg[g].data_ptr(), 24, table,
                                                                                        sp_dg[g].data_ptr(), pd_dg[g].data_ptr())
                                        if v == "c":
                                            copy(drv.cuMemcpyDtoHAsync_v2, sp_hg[g], sp_dg[g], s)
                                            copy(drv.cuMemcpyDtoHAsync_v2, pd_hg[g], pd_dg[g], s)
                                    if r >= a.warmup:
                                        host.append((time.perf_counter() - t0) * 1e3)
                                for ln in lanes:
                                    eng.lane_sync(ln)
                            out[v + "_round_ms"] = round((time.perf_counter() - t_start) * 1e3 / a.rounds, 3)
                            if v in "ad":
                                out[v + "_call_host_ms_median"] = round(float(np.median(host)), 4)
                        bytes_in = G * n * F * 6
                        bytes_out = G * n * F * (P * w * 4 + 32)
                        out["link_ms"] = round(max(bytes_in / (bw["h2d"] * 1e9), bytes_out / (bw["d2h"] * 1e9)) * 1e3, 3)
                        out["bound_ms"] = max(out["link_ms"], out["b_round_ms"])
                        out.update(info)
                        print(json.dumps(out), flush=True)
                    finally:
                        for ln in lanes:
                            eng.lane_close(ln)
    finally:
        eng.close()


def run():
    import torch

    assert torch.cuda.is_available(), "chain_lane_host_bench needs a GPU"
    info = card(torch)
    info["max_connections"] = os.environ.get("CUDA_DEVICE_MAX_CONNECTIONS", "default (8)")
    bw = link(torch)
    info["h2d_GBps"], info["d2h_GBps"] = round(bw["h2d"], 2), round(bw["d2h"], 2)
    for arith in a.ariths.split(","):
        run_arith(arith, info, bw)


if __name__ == "__main__":
    if a.child:
        run()
    else:
        for k in a.connections.split(","):
            env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS=k)
            args = [sys.executable, os.path.abspath(__file__), "--child", "--ariths", a.ariths, "--groups", a.groups, "--sizes", a.sizes,
                    "--forms", a.forms, "--rounds", str(a.rounds), "--warmup", str(a.warmup)]
            subprocess.check_call(args, env=env)
