#!/usr/bin/env python
"""What an instance-range process call costs next to a whole-engine call, on one engine of 8192 instances.
    python scripts/chain_range_bench.py [--instances 8192] [--packets 64] [--fpp 96] [--reps 20] [--parent DIR] [--rounds 3]

For the float fused and the Q28 chain, words output (BASELINE config 3 parameters): a whole-engine call through
dspi_chain(q)_process_packets_device, then dspi_chain(q)_process_packets_range_device over [0, n) for n = 4096, 1024, 256
and 64, each with buffers of its own n rows.  Times are CUDA events on the engine stream around --reps calls after a
warm-up call, in ms per call.  Range time falls with n down to a floor set by the launches of a call: per packet slice a
range call launches K1 / K2 once per role (11 float, 7 Q28) where a whole-engine call launches it twice, and the
modulator is one serial chain per instance whatever n is.  Each set runs twice: as configured (sub on), and with the sub
output disabled, which leaves the modulator idle and shows what the other stages cost at each n.

--parent DIR: a checkout of another revision with its library built; its scripts/chain_bench.py and this tree's run the
same whole-engine workload in alternation, --rounds times each, so that the two revisions are compared in one session.
Every result line carries the card name and power limit it was measured at."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np                                        # noqa: E402
import torch                                              # noqa: E402
from dspi_b200 import api, workloads as W                  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--instances", type=int, default=8192)
ap.add_argument("--packets", type=int, default=64)
ap.add_argument("--fpp", type=int, default=96)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--sizes", default="4096,1024,256,64")
ap.add_argument("--parent", default=None)
ap.add_argument("--rounds", type=int, default=3)
a = ap.parse_args()


def card():
    """name and power limit of device 0, read in the same run as the numbers"""
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        limit = q.stdout.strip() if q.returncode == 0 else "unknown"
    except (OSError, subprocess.TimeoutExpired):
        limit = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": limit}


def timed(eng, step, reps):
    step()
    eng.sync()
    st = torch.cuda.ExternalStream(eng.stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(reps):
        step()
    e1.record(st)
    eng.sync()
    return e0.elapsed_time(e1) / reps


def ranges(arith, info, sub_on):
    N, F, fs = a.instances, a.packets * a.fpp, 96000.0
    q28 = arith == "q28"
    if q28:
        P, bq = W.chain_config3_q28(N, fs=fs)
        eng = api.ChainEngineQ28(N, max_frames=F)
    else:
        P, bq = W.chain_config3(N, fs=fs, seed=1)
        eng = api.ChainEngine(arith, N, max_frames=F)
    if not sub_on:                                        # no modulator work: what the other stages cost at each n
        P["matrix"]["outputs"]["enabled"][:, (5 if q28 else 9) - 1] = 0
    try:
        eng.set_params(P)
        eng.upload_biquads(bq)
        pairs = 2 if q28 else 4
        table = np.full(a.packets, a.fpp, np.uint16)
        pcm = torch.randint(0, 256, (N, F * 6), dtype=torch.uint8, device="cuda")
        spdif = torch.empty((N, pairs, F, 2), dtype=torch.int32, device="cuda")
        pdm = torch.empty((N, F, 8), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        out = {"arith": arith, "sub": sub_on, "instances": N, "packets": a.packets, "fpp": a.fpp, "reps": a.reps, **info}
        l0 = eng.launch_count
        out["whole_ms"] = timed(eng, lambda: eng.process_packets_device(pcm.data_ptr(), 24, table, spdif.data_ptr(), pdm.data_ptr()), a.reps)
        out["whole_launches_per_call"] = (eng.launch_count - l0) / (a.reps + 1)
        for n in (int(s) for s in a.sizes.split(",")):
            # own n-row buffers, as a host serving one device group would hold
            sp, pd = torch.empty((n, pairs, F, 2), dtype=torch.int32, device="cuda"), torch.empty((n, F, 8), dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            l0 = eng.launch_count
            out[f"range_{n}_ms"] = timed(eng, lambda: eng.process_packets_range_device(0, n, pcm.data_ptr(), 24, table, sp.data_ptr(), pd.data_ptr()), a.reps)
            out[f"range_{n}_launches_per_call"] = (eng.launch_count - l0) / (a.reps + 1)
        print(json.dumps(out), flush=True)
    finally:
        eng.close()


def whole_engine_ab(info):
    """this tree and --parent in alternation on scripts/chain_bench.py's whole-engine workload"""
    res = {}
    for arith in ("f32f", "q28"):
        for r in range(a.rounds):
            for tag, tree in (("parent", os.path.abspath(a.parent)), ("branch", ROOT)):
                cmd = [sys.executable, os.path.join(tree, "scripts", "chain_bench.py"), "--arith", arith, "--instances", str(a.instances),
                       "--packets", str(a.packets), "--fpp", str(a.fpp), "--reps", str(a.reps)]
                p = subprocess.run(cmd, capture_output=True, text=True, cwd=tree)
                if p.returncode != 0:
                    raise RuntimeError(f"{tag} {arith}: {p.stderr[-2000:]}")
                ms = json.loads(p.stdout.strip().splitlines()[-1])["ms_per_step"]
                res.setdefault(f"{arith}_{tag}_ms", []).append(ms)
    for arith in ("f32f", "q28"):
        for tag in ("parent", "branch"):
            v = res[f"{arith}_{tag}_ms"]
            res[f"{arith}_{tag}_median_ms"] = float(np.median(v))
    print(json.dumps({"whole_engine_ab": res, "packets": a.packets, "fpp": a.fpp, "instances": a.instances, **info}), flush=True)


if __name__ == "__main__":
    assert torch.cuda.is_available(), "chain_range_bench needs a GPU"
    info = card()
    for sub_on in (True, False):
        for arith in ("f32f", "q28"):
            ranges(arith, info, sub_on)
    if a.parent:
        whole_engine_ab(info)
