"""Times dspi_chain(q)_copy_instances against the host image route it replaces, on 8192-instance float (fused) and Q28
engines, in one run:

  copy       one copy_instances call of n scattered pairs (n = 1, 64, 900, 4096; distinct random sources and destinations),
             on a host clock (the call ends in a synchronise), median of --reps calls
  host loop  the same pairs through export_instances(src[k], 1) then import_instances(dst[k], 1), per pair, on a host clock
  kernel     in a profiled call of its own, the device time of the copy kernel (instance_copy_kernel) and of everything
             else the call runs (EQ unpack / pack, skip masks, list and envelope-mode copies); the kernel's bytes moved
             (every image byte of each pair read once and written once, header excluded) per second, against the H100 SXM
             data-sheet HBM3 peak

The engines are configured (set_params + biquads) and have run one call, so the instances hold non-trivial data.  Prints
the card, its power limit and max SM clock, read in the same run, then one JSON line per engine kind and n.  Fails without
a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from instance_image_bench import HBM_PEAK, configured, host_clock     # noqa: E402

HEADER = 32                                                   # bytes of an image that the copy does not move


def device_split(call):
    """device time (s) of the copy kernel and of everything else in one call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    out = {"kernel": 0.0, "other": 0.0, "kernel_launches": 0}
    for ev in prof.key_averages():
        t = (getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)) * 1e-6
        if "instance_copy_kernel" in ev.key:
            out["kernel"] += t
            out["kernel_launches"] += ev.count
        elif t > 0:
            out["other"] += t
    return out


def host_loop(eng, src, dst):
    for s, d in zip(src, dst):
        eng.import_instances(eng.export_instances(int(s), 1), inst0=int(d))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--loop-reps", type=int, default=2)
    ap.add_argument("--pairs", type=int, nargs="+", default=[1, 64, 900, 4096])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("copy_instances_bench: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))
    N = a.instances
    rng = np.random.default_rng(7)
    for kind in ("f32f", "q28"):
        eng = configured(kind, N)
        size = eng.instance_image_size()
        for n in a.pairs:
            perm = rng.permutation(N)
            src, dst = perm[:n].astype(np.uint32), perm[n:2 * n].astype(np.uint32)
            eng.copy_instances(src, dst)                                # warm-up
            host_loop(eng, src[:1], dst[:1])
            t_copy = host_clock(lambda: eng.copy_instances(src, dst), a.reps)
            t_loop = host_clock(lambda: host_loop(eng, src, dst), a.loop_reps)
            s = device_split(lambda: eng.copy_instances(src, dst))
            moved = 2.0 * n * (size - HEADER)
            out = {"case": f"{kind} {N} instances, {n} pairs", "image_bytes": size, "bytes_moved": int(moved),
                   "copy_ms": round(float(np.median(t_copy)) * 1e3, 3), "host_loop_ms": round(float(np.median(t_loop)) * 1e3, 2),
                   "kernel_ms": round(s["kernel"] * 1e3, 4), "kernel_launches": s["kernel_launches"], "other_device_ms": round(s["other"] * 1e3, 4),
                   "kernel_GBps": round(moved / s["kernel"] / 1e9, 1) if s["kernel"] else None,
                   "kernel_share_of_hbm_peak": round(moved / s["kernel"] / HBM_PEAK, 3) if s["kernel"] else None}
            print(json.dumps(out), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
