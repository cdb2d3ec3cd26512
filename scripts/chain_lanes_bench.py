#!/usr/bin/env python
"""What lanes buy: G clock groups of n instances served by G sequential range calls on the engine stream, against one call
per group on lanes of their own (dspi_chain(q)_lane_*), on one engine of 8192 instances.
    python scripts/chain_lanes_bench.py [--groups 1,2,4,8] [--sizes 64,256,1024] [--reps 5] [--trace-dir DIR]

For the float fused and the Q28 chain (BASELINE config 3 parameters, 96 kHz, words and PDM output), sub output on and off.
Group g covers instances [g n, (g + 1) n) with its own packet table: "64x96" gives every group 64 packets of 96 frames,
"cadence" gives the odd groups the 10-packet 44.1 kHz cadence (9 x 44 + 45 frames) instead.  A round is one call per
group followed by dspi_chain_sync (which waits for the lanes); it is timed with the host clock around the whole round.  After
a warm-up round, the two modes run alternately five times each and the best of each is reported, in ms per round.

Before timing, each configuration checks that both modes give byte-identical words and PDM: two more engines, configured
alike and given the same rounds throughout, run one round each, one as sequential range calls and one on lanes.  The "edit" variant adds one
dspi_chain(q)_edit_bulk_device call per round before the group calls (instances configured through set_params, which the
call reports as stale and leaves alone; it still joins every lane and runs its upload and kernel), which prices the
barrier an engine-level call puts across the lanes.

A separate torch.profiler run (G = 4, n = 256, float, sub on) counts, for each mode, the most modulator kernels in flight
at once and the streams the kernels ran on: with lanes, modulator kernels of different groups overlap.  Every result line
carries the card name, power limit and max SM clock it was measured at."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np                                        # noqa: E402
import torch                                              # noqa: E402
from dspi_b200 import api, layouts as L, workloads as W    # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--instances", type=int, default=8192)
ap.add_argument("--groups", default="1,2,4,8")
ap.add_argument("--sizes", default="64,256,1024")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--trace-dir", default=None)
a = ap.parse_args()
CADENCE = [44] * 9 + [45]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        limit = q.stdout.strip() if q.returncode == 0 else "unknown"
    except (OSError, subprocess.TimeoutExpired):
        limit = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": limit}


def make_engine(arith, sub_on, F):
    N, fs = a.instances, 96000.0
    q28 = arith == "q28"
    if q28:
        P, bq = W.chain_config3_q28(N, fs=fs)
        eng = api.ChainEngineQ28(N, max_frames=F)
    else:
        P, bq = W.chain_config3(N, fs=fs, seed=1)
        eng = api.ChainEngine(arith, N, max_frames=F)
    if not sub_on:
        P["matrix"]["outputs"]["enabled"][:, (5 if q28 else 9) - 1] = 0
    eng.set_params(P)
    eng.upload_biquads(bq)
    return eng, (2 if q28 else 4)


class Groups:
    """G groups of n instances, each with its table, its input rows and its output buffers, and a lane per group"""

    def __init__(self, eng, pairs, G, n, sched, pcm):
        self.eng, self.G, self.n = eng, G, n
        self.tables = [np.array(CADENCE if sched == "cadence" and g % 2 else [96] * 64, np.uint16) for g in range(G)]
        self.row = pcm.shape[1]
        self.pcm = pcm
        self.out = [(torch.zeros((n, pairs, int(t.sum()), 2), dtype=torch.int32, device="cuda"),
                     torch.zeros((n, int(t.sum()), 8), dtype=torch.int32, device="cuda")) for t in self.tables]
        torch.cuda.synchronize()
        self.lanes = [eng.lane_open(g * n, n) for g in range(G)]
        self.edit = np.concatenate([L.bulk_edit(g * n, ("outputs", 0, "gain_db"), np.float32(-1.0)) for g in range(G)])

    def close(self):
        for ln in self.lanes:
            self.eng.lane_close(ln)

    def round(self, lanes, edit=False):
        e = self.eng
        if edit:
            e.edit_bulk_device(self.edit, 96000.0)
        for g, (t, (sp, pd)) in enumerate(zip(self.tables, self.out)):
            args = (g * self.n, self.n, self.pcm.data_ptr() + g * self.n * self.row, 24, t, sp.data_ptr(), pd.data_ptr())
            if lanes:
                e.lane_process_packets_device(self.lanes[g], *args)
            else:
                e.process_packets_range_device(*args)
        e.sync()

    def outputs(self):
        return [(sp.cpu().numpy().copy(), pd.cpu().numpy().copy()) for sp, pd in self.out]


def same_outputs(seq, lan):
    seq.round(False)
    lan.round(True)
    return all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(seq.outputs(), lan.outputs()))


def timed(gr, edit):
    gr.round(False, edit)
    gr.round(True, edit)
    best = {False: float("inf"), True: float("inf")}
    for _ in range(a.reps):
        for lanes in (False, True):
            t0 = time.perf_counter()
            gr.round(lanes, edit)
            best[lanes] = min(best[lanes], (time.perf_counter() - t0) * 1e3)
    return best[False], best[True]


def sweep(info):
    F = 64 * 96
    groups, sizes = [int(x) for x in a.groups.split(",")], [int(x) for x in a.sizes.split(",")]
    for arith in ("f32f", "q28"):
        for sub_on in (True, False):
            eng, pairs = make_engine(arith, sub_on, F)
            twins = [make_engine(arith, sub_on, F)[0] for _ in range(2)]
            pcm = torch.randint(0, 256, (a.instances, F * 6), dtype=torch.uint8, device="cuda")
            try:
                for sched in ("64x96", "cadence"):
                    for n in sizes:
                        for G in groups:
                            if G * n > a.instances or (sched == "cadence" and G == 1):
                                continue
                            gr = Groups(eng, pairs, G, n, sched, pcm)
                            check = [Groups(e, pairs, G, n, sched, pcm) for e in twins]
                            try:
                                out = {"arith": arith, "sub": sub_on, "sched": sched, "G": G, "n": n, "identical": same_outputs(*check),
                                       "max_connections": os.environ.get("CUDA_DEVICE_MAX_CONNECTIONS", "default"), **info}
                                out["seq_ms"], out["lanes_ms"] = timed(gr, False)
                                out["speedup"] = out["seq_ms"] / out["lanes_ms"]
                                if sched == "64x96" and n == 256 and G in (2, 4):
                                    out["seq_edit_ms"], out["lanes_edit_ms"] = timed(gr, True)
                                print(json.dumps(out), flush=True)
                            finally:
                                for x in [gr] + check:
                                    x.close()
            finally:
                for e in [eng] + twins:
                    e.close()


def overlap(trace):
    """most modulator kernels in flight at once, and the number of streams kernels ran on"""
    ev = json.load(open(trace))["traceEvents"]
    ks = [e for e in ev if e.get("cat") == "kernel"]
    pdm = sorted((e["ts"], e["ts"] + e["dur"]) for e in ks if "pdm_kernel" in e["name"])
    edges = sorted([(s, 1) for s, _ in pdm] + [(t, -1) for _, t in pdm], key=lambda x: (x[0], x[1]))
    cur = best = 0
    for _, d in edges:
        cur += d
        best = max(best, cur)
    return best, len({e["args"].get("stream") for e in ks})


def profile(info):
    F = 64 * 96
    eng, pairs = make_engine("f32f", True, F)
    pcm = torch.randint(0, 256, (a.instances, F * 6), dtype=torch.uint8, device="cuda")
    gr = Groups(eng, pairs, 4, 256, "64x96", pcm)
    d = a.trace_dir or tempfile.mkdtemp()
    os.makedirs(d, exist_ok=True)
    out = {"profile": "G=4 n=256 f32f sub on 64x96", **info}
    try:
        for lanes in (False, True):
            gr.round(lanes)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    gr.round(lanes)
            path = os.path.join(d, "lanes_%s.json" % ("on" if lanes else "off"))
            prof.export_chrome_trace(path)
            out["lanes" if lanes else "seq"] = dict(zip(("max_modulators_in_flight", "kernel_streams"), overlap(path)))
    finally:
        gr.close()
        eng.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    assert torch.cuda.is_available(), "chain_lanes_bench needs a GPU"
    info = card()
    sweep(info)
    profile(info)
