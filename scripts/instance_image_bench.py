"""Times the per-instance lifecycle calls of both chain engines (dspi_chain(q)_export_instances / _import_instances /
_reset_instances), in one run:

  bulk         export and import of every instance of an 8192-instance float (fused) and Q28 engine: the call on a host
               clock (it ends in a device synchronise), and in a profiled call of its own the device time of the copy
               kernel (instance_image_kernel, all chunks) against the host <-> device copies, with the kernel's bytes moved
               (every image byte read once and written once) per second against the H100 SXM data-sheet HBM3 peak
  one          export, import and reset of ONE instance on engines of 64 and 8192 instances (median of many calls)
  state_export the whole-engine checkpoint of the same 8192-instance engine, for comparison

The engines are configured (set_params + biquads) and have run one call, so the images hold non-trivial data.  Images and
blobs live in ordinary (pageable) host memory, as the Python API returns them.  Prints the card, its power limit and max SM
clock, read in the same run, then one JSON line per engine kind.  Fails without a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dspi_b200 import api, layouts as L, workloads as W     # noqa: E402

FS = 48000.0
HBM_PEAK = 3.35e12                                           # H100 SXM data sheet, bytes/s


def host_clock(call, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()
        ts.append(time.perf_counter() - t0)
    return ts


def device_split(call):
    """device time (s) of the image kernel, of the host <-> device copies and of everything else in one call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    out = {"kernel": 0.0, "copy": 0.0, "other": 0.0, "kernel_launches": 0}
    for ev in prof.key_averages():
        t = (getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)) * 1e-6
        if "instance_image_kernel" in ev.key:
            out["kernel"] += t
            out["kernel_launches"] += ev.count
        elif ev.key.startswith("Memcpy"):
            out["copy"] += t
        elif t > 0:
            out["other"] += t
    return out


def configured(kind, n):
    q28 = kind == "q28"
    eng = api.ChainEngineQ28(n, 192) if q28 else api.ChainEngine(kind, n, 192)
    roles = L.CHAINQ_EQ_CHANNELS if q28 else L.CHAIN_EQ_CHANNELS
    P = np.zeros(n, L.CHAIN_PARAMS_Q28 if q28 else L.CHAIN_PARAMS_F32)
    P["leveller_enabled"], P["leveller_lookahead"] = 1, 1
    for o in range(5 if q28 else 9):
        P["matrix"]["outputs"][:, o]["enabled"] = 1
        P["matrix"]["outputs"][:, o]["delay_samples"] = 37 * o
        P["matrix"]["crosspoints"][:, 0, o]["enabled"] = 1
    eng.set_params(P)
    bq = api.compute_coefficients(W.eq_params("B", roles, fs=FS, seed=1), q28=q28, fs=FS)
    eng.upload_biquads(np.broadcast_to(bq, (n, roles, L.MAX_BANDS)))
    rng = np.random.default_rng(2)
    eng.process_packets_host(rng.integers(0, 256, (n, 192 * 6), dtype=np.uint8), 24, [96, 96], want_spdif=False, want_pdm=False)
    return eng


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--one-reps", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("instance_image_bench: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))
    N = a.instances
    for kind in ("f32f", "q28"):
        eng = configured(kind, N)
        size = eng.instance_image_size()
        img = eng.export_instances()                                   # warm-up of both directions
        eng.import_instances(img)
        exp = host_clock(lambda: eng.export_instances(), a.reps)
        imp = host_clock(lambda: eng.import_instances(img), a.reps)
        split_e = device_split(lambda: eng.export_instances())
        split_i = device_split(lambda: eng.import_instances(img))
        moved = 2.0 * size * N
        eng.state_export()
        st = host_clock(lambda: eng.state_export(), a.reps)
        out = {"case": f"{kind} {N} instances", "image_bytes": size, "state_blob_bytes": int(eng._fn("state_size")(eng._h)),
               "export_ms": round(min(exp) * 1e3, 2), "import_ms": round(min(imp) * 1e3, 2), "state_export_ms": round(min(st) * 1e3, 2)}
        for name, s in (("export", split_e), ("import", split_i)):
            out[name + "_device"] = {"kernel_ms": round(s["kernel"] * 1e3, 3), "kernel_launches": s["kernel_launches"],
                                     "copy_ms": round(s["copy"] * 1e3, 2), "other_ms": round(s["other"] * 1e3, 3),
                                     "kernel_GBps": round(moved / s["kernel"] / 1e9, 1) if s["kernel"] else None,
                                     "kernel_share_of_hbm_peak": round(moved / s["kernel"] / HBM_PEAK, 3) if s["kernel"] else None,
                                     "kernel_over_copy": round(s["kernel"] / s["copy"], 4) if s["copy"] else None}
        one = {}
        small = configured(kind, 64)
        for label, e in (("n64", small), (f"n{N}", eng)):
            i1 = e.export_instances(7, 1)
            for _ in range(3):
                e.export_instances(7, 1); e.import_instances(i1, 7); e.reset_instances(7, 1)   # noqa: E702
            one[label] = {k: round(float(np.median(host_clock(c, a.one_reps))) * 1e6, 1) for k, c in
                          (("export_us", lambda: e.export_instances(7, 1)), ("import_us", lambda: e.import_instances(i1, 7)),
                           ("reset_us", lambda: e.reset_instances(7, 1)))}
        out["one_instance_median"] = one
        small.close()
        eng.close()
        print(json.dumps(out))


if __name__ == "__main__":
    main()
