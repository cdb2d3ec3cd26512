#!/usr/bin/env python
"""BASELINE config 3 alone: N instances through the whole chain, device-resident, CUDA events.
    python scripts/chain_bench.py [--instances 8192] [--packets 16] [--fpp 96] [--reps 3] [--schedule uniform|44k1|feedback]
                                  [--spdif words|encode|subframes]

--schedule picks the packet lengths of a call: `uniform` is --packets packets of --fpp frames at 96 kHz through
dspi_chain(q)_process_device; `44k1` is the 44.1 kHz cadence (nine 44-frame packets, then one of 45) at fs = 44100, and
`feedback` seeded lengths in {95, 96, 97} at 96 kHz (an asynchronous device's feedback pacing), both through
dspi_chain(q)_process_packets_device.  The real-time factor uses the schedule's own sample rate.

--spdif picks the S/PDIF output: `words` is the 24-bit words form alone; `encode` is the words form followed by
dspi_spdif_encode_device over those words on the engine stream (the two-pass path to the wire format); `subframes` is
dspi_chain(q)_process_subframes_device, whose output stage writes the subframes itself.  The JSON line names the mode and
the bytes of the output buffers it writes."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np                                        # noqa: E402
import torch                                              # noqa: E402
from dspi_b200 import api, workloads as W                  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--instances", type=int, default=8192)
ap.add_argument("--packets", type=int, default=16)
ap.add_argument("--fpp", type=int, default=96)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--arith", default="f32f")
ap.add_argument("--no-sub", action="store_true", help="disable the sub output: no modulator work (isolates the other stages)")
ap.add_argument("--schedule", choices=["uniform", "44k1", "feedback"], default="uniform")
ap.add_argument("--spdif", choices=["words", "encode", "subframes"], default="words")
a = ap.parse_args()
if a.schedule == "uniform":
    frames, fs = None, 96000.0
elif a.schedule == "44k1":
    frames, fs = np.resize(np.array([44] * 9 + [45], np.uint16), a.packets), 44100.0
else:
    frames, fs = np.random.default_rng(1).integers(95, 98, a.packets).astype(np.uint16), 96000.0
N = a.instances
F = a.packets * a.fpp if frames is None else int(frames.sum())
q28 = a.arith == "q28"
if q28:
    P, bq = W.chain_config3_q28(N, fs=fs)
    eng = api.ChainEngineQ28(N, max_frames=F)
else:
    P, bq = W.chain_config3(N, fs=fs, seed=1)
    eng = api.ChainEngine(a.arith, N, max_frames=F)
n_out = 5 if q28 else 9
if a.no_sub:
    P["matrix"]["outputs"]["enabled"][:, n_out - 1] = 0
eng.set_params(P)
eng.upload_biquads(bq)
pairs = 2 if q28 else 4
pcm = torch.randint(0, 256, (N, F * 6), dtype=torch.uint8, device="cuda")
spdif = torch.empty((N, pairs, F, 2), dtype=torch.int32, device="cuda") if a.spdif != "subframes" else None
sub = torch.empty((N, pairs, F, 2, 2), dtype=torch.int32, device="cuda") if a.spdif != "words" else None
pdm = torch.empty((N, F, 8), dtype=torch.int32, device="cuda")
torch.cuda.synchronize()
table = np.full(a.packets, a.fpp, np.uint16) if frames is None else frames


def step():
    if a.spdif == "subframes":
        eng.process_subframes_device(pcm.data_ptr(), 24, table, sub.data_ptr(), pdm.data_ptr())
        return
    if frames is None:
        eng.process_device(pcm.data_ptr(), 24, a.packets, a.fpp, spdif.data_ptr(), pdm.data_ptr())
    else:
        eng.process_packets_device(pcm.data_ptr(), 24, frames, spdif.data_ptr(), pdm.data_ptr())
    if a.spdif == "encode":
        api.spdif_encode_device(spdif.data_ptr(), N * pairs, F, sub.data_ptr(), device=eng.device, stream=eng.stream)


step()
eng.sync()
if q28:                                                   # no stream accessor on the Q28 chain: host clock around synchronised calls
    import time
    t0 = time.perf_counter()
    for _ in range(a.reps):
        step()
    eng.sync()
    ms = (time.perf_counter() - t0) * 1e3 / a.reps
else:
    st = torch.cuda.ExternalStream(eng.stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(a.reps):
        step()
    e1.record(st)
    eng.sync()
    ms = e0.elapsed_time(e1) / a.reps
print(json.dumps({"schedule": a.schedule, "packets": a.packets, "fs": fs, "instances": N, "frames": F, "sm_partition": eng.sm_partition(),
                  "spdif": a.spdif, "output_bytes": {"words": spdif.nbytes if spdif is not None else 0, "subframes": sub.nbytes if sub is not None else 0,
                                                     "pdm": pdm.nbytes},
                  "ms_per_step": ms, "instance_frames_per_s": N * F / (ms * 1e-3),
                  "arith": a.arith, "output_channel_samples_per_s": N * n_out * F / (ms * 1e-3), "realtime_factor": (F / fs) / (ms * 1e-3)}))
