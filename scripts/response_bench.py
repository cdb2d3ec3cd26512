"""Times the frequency-response kernels with CUDA events after warm-up:
dspi_eq_response_device at 65 536 channels x 10 bands x 1024 frequencies (float and Q28) and both chain responses at
8192 instances x 1024 frequencies.  Prints the card and its power limit, read in the same run, and for each shape the
FP64 operations and bytes computed from the shape and the share of the binding bound.

FP64 operations per (row, frequency, active band): 14 for the section (two quadratics in w) + 12 for the two complex
products = 26, plus 11 for the complex division per row.  Bytes: the float2 output; reads are negligible.
Peaks (H100 SXM data sheet, 700 W): FP64 34 TFLOP/s (non-tensor), HBM3 3.35 TB/s."""
import argparse
import json
import subprocess
import sys
import os

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dspi_b200 import api, layouts as L, workloads as W     # noqa: E402

FP64_PEAK, HBM_PEAK = 34e12, 3.35e12


def timed(fn, stream, reps, warmup):
    """Seconds per call; the events are recorded on the engine's own stream, where the calls run."""
    import torch
    s = torch.cuda.ExternalStream(stream)
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(s)
    for _ in range(reps):
        fn()
    b.record(s)
    b.synchronize()
    return a.elapsed_time(b) / reps * 1e-3


def report(name, sec, flops, nbytes):
    t_f, t_b = flops / FP64_PEAK, nbytes / HBM_PEAK
    bound = "FP64" if t_f >= t_b else "HBM"
    r = {"case": name, "ms": round(sec * 1e3, 4), "gflop": round(flops / 1e9, 2), "mbytes": round(nbytes / 1e6, 1),
         "fp64_tflops": round(flops / sec / 1e12, 2), "gbytes_s": round(nbytes / sec / 1e9, 1),
         "bound": bound, "fraction_of_bound": round(max(t_f, t_b) / sec, 3)}
    print(json.dumps(r))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--freqs", type=int, default=1024)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))
    fs = 48000.0
    f = np.geomspace(10.0, 23990.0, a.freqs).astype(np.float32)
    nf = f.size
    C = 65536
    for arith in ("f32f", "q28"):
        e = api.EqEngine(arith, C)
        e.set_params_device(W.eq_params_fast("B", C, fs=fs, seed=1), fs)
        active = int(np.sum(e.download()["bypass"][:, :10] == 0))
        out = torch.empty((C, nf), dtype=torch.complex64, device="cuda")
        sec = timed(lambda: e.response(f, fs, out_ptr=out.data_ptr()), e.stream, a.reps, a.warmup)
        report(f"eq {arith} {C} ch x 10 bands x {nf} f", sec, (26.0 * active + 11.0 * C) * nf, C * nf * 8.0)
        e.close()
    N = 8192
    for arith in ("f32f", "q28"):
        if arith == "q28":
            P, bq = W.chain_config3_q28(N, fs=fs)
            ce = api.ChainEngineQ28(N, 192)
        else:
            P, bq = W.chain_config3(N, fs=fs)
            ce = api.ChainEngine(arith, N, 192)
        ce.set_params(P)
        ce.upload_biquads(bq)
        rows = bq.shape[1]
        active = int(np.sum(bq["bypass"][:, :, :10] == 0))
        outs = rows - 2
        out = torch.empty((N, outs, 2, nf), dtype=torch.complex64, device="cuda")
        sec = timed(lambda: ce.response(f, fs, out_ptr=out.data_ptr()), ce.stream, a.reps, a.warmup)
        # sections and row divisions as for the EQ; crossfeed, delays and the 2 x outputs combinations about 200 more per instance
        report(f"chain {arith} {N} inst x {nf} f", sec, (26.0 * active + 11.0 * rows * N + 200.0 * N) * nf, N * outs * 2 * nf * 8.0)
        ce.close()


if __name__ == "__main__":
    main()
