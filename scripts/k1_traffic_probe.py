#!/usr/bin/env python
"""Where K1's headline step spends its time: the float EQ cascade at bench.py's shape (65 536 channels x 6144 samples,
fused, variant A), timed in three modes on one engine:
    full    the kernel as shipped
    dbg1    DSPI_DBG=1: the data path only (TMA loads, shared-memory shuffles, TMA stores), no filter arithmetic
    dbg2    DSPI_DBG=2: the arithmetic only, no HBM traffic
Each mode is timed with CUDA events over --steps launches after --warmup, rotating over buffers larger than L2.
The geometry is the one the engine picks from the environment (DSPI_F32_CPL).  Prints one JSON line.
    python scripts/k1_traffic_probe.py [--steps 30] [--warmup 5]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dspi_b200 import api, workloads as W          # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--channels", type=int, default=65536)
ap.add_argument("--frames", type=int, default=6144)
ap.add_argument("--steps", type=int, default=30)
ap.add_argument("--warmup", type=int, default=5)
a = ap.parse_args()
FS = 96000.0
C, T = a.channels, a.frames

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                           str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                    # the numbers stand without it, but say why it is missing
    card = f"nvidia-smi unavailable: {e!r}"

eng = api.EqEngine("f32f", C)
eng.upload(api.compute_coefficients(W.eq_params_fast("A", C, fs=FS, seed=1), fs=FS))
nbuf = 4                                                  # 4 x 1.5 GiB, each far larger than the 50 MB L2
bufs = [torch.rand((C, T), dtype=torch.float32, device="cuda") - 0.5 for _ in range(nbuf)]
torch.cuda.synchronize()
st = torch.cuda.ExternalStream(eng.stream)
saved = os.environ.get("DSPI_DBG")
res = {"card": card, "kernel_variant": eng.kernel_info(), "channels": C, "frames": T, "steps": a.steps,
       "env": {"DSPI_F32_CPL": os.environ.get("DSPI_F32_CPL")}, "modes": {}}
for mode, dbg in (("full", None), ("dbg1", "1"), ("dbg2", "2")):
    if dbg is None:
        os.environ.pop("DSPI_DBG", None)
    else:
        os.environ["DSPI_DBG"] = dbg                      # read by the engine at every launch
    for i in range(a.warmup):
        eng.process_device(bufs[i % nbuf].data_ptr(), T, T)
    eng.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for i in range(a.steps):
        eng.process_device(bufs[i % nbuf].data_ptr(), T, T)
    e1.record(st)
    eng.sync()
    ms = e0.elapsed_time(e1) / a.steps
    # algorithmic traffic: 4 B read + 4 B written per channel-sample (bench.py); the dbg2 mode moves none of it
    res["modes"][mode] = {"ms_per_step": ms, "GB_s": C * T * 8 / (ms * 1e-3) / 1e9, "G_samples_s": C * T / (ms * 1e-3) / 1e9}
if saved is None:
    os.environ.pop("DSPI_DBG", None)
else:
    os.environ["DSPI_DBG"] = saved
print(json.dumps(res))
eng.close()
