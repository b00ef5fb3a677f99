"""What the reference arithmetic (PWPP_ARITH_REFERENCE: sequential fp32 plane fits, csrc/pwpp_fit_ref32.cuh) costs over the default
double arithmetic. One JSON line per record on stdout and in --out. Run on the GPU from the repository root after build():

  python tools/ref32_bench.py [--steps K] [--reps R] [--out FILE]

  gpu       card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  batch     step time of one pwpp_estimate_device call over 1024 frames resident in HBM (every frame on a fresh stream), for
            bench.py's synthetic KITTI-64 batch and for the six recorded KITTI scans cycled to 1024 frames; the two modes
            alternate, R rounds of K steps each (CUDA events); with the per-stage device times of one profiled step of each mode
            (the fit classes then run one after another) and the largest patch of the batch
  drop_in   one-frame latency of the drop-in class's pattern (estimateGround + both index getters: upload, kernels, lists back on
            the host) over the six recorded scans, both modes alternating, wall clock, with the stage times of one profiled call
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, "patchwork-plusplus_b200")
for p in (PKG, os.path.join(PKG, "lib"), REPO):
    if p not in sys.path:
        sys.path.insert(0, p)

MODES = {"double": 0, "reference": 1}


def gpu_info():
    q = "name,power.limit,clocks.max.sm,driver_version"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, clk, drv = [x.strip() for x in out[0].split(",")]
    return {"record": "gpu", "name": name, "power_limit": plim, "max_sm_clock": clk, "driver": drv}


def kitti():
    return [np.ascontiguousarray(np.load(os.path.join(REPO, "tests", "golden", f"kitti_{k:06d}.npz"))["xyzi_t"].T, dtype=np.float32) for k in range(6)]


def batch(workload, steps, reps):
    import torch
    import bench
    import pwpp_b200
    import synth
    F = 1024
    dev = torch.device("cuda", 0)
    if workload == "synthetic":
        pts, offs = synth.make_batch(bench.SEED, 0, F, "kitti64", dev)
        offs_np = offs.numpy()
    else:
        fr = kitti()
        a = np.concatenate([fr[f % 6] for f in range(F)])
        offs_np = np.r_[0, np.cumsum([len(fr[f % 6]) for f in range(F)])].astype(np.int64)
        pts = torch.from_numpy(a).to(dev)
    ts = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(ts)
    engs = {}
    for name, mode in MODES.items():
        e = pwpp_b200.Engine(device=0, num_streams=F, max_points_per_frame=int(np.diff(offs_np).max()))
        e.set_arithmetic(mode)
        engs[name] = e

    def step(e):
        e.reset()
        e.estimate_device(pts.data_ptr(), offs_np, True, ts.cuda_stream)
    out = {"record": "batch", "workload": workload, "frames": F, "points": int(offs_np[-1]), "steps": steps, "rounds": reps}
    for name, e in engs.items():   # warm-up, then one profiled step: per-stage device times
        for _ in range(3):
            step(e)
        torch.cuda.synchronize()
        e.set_profiling(True)
        step(e)
        out[f"stage_ms_{name}"] = e.stage_times_ms()
        e.set_profiling(False)
        if name == "reference":
            out["largest_patch_points"] = max(max(r.n for r in e.bin_results(f)) for f in range(0, F, 64))
    times = {k: [] for k in engs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(reps):
        for name, e in engs.items():
            e0.record(ts)
            for _ in range(steps):
                step(e)
            e1.record(ts)
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / steps)
    for name, e in engs.items():
        l0 = e.launch_count(); step(e); torch.cuda.synchronize()
        out[f"launches_per_step_{name}"] = e.launch_count() - l0
        out[f"ms_per_step_{name}"] = float(np.median(times[name]))
        out[f"ms_per_step_{name}_runs"] = times[name]
        e.close()
    out["reference_over_double"] = out["ms_per_step_reference"] / out["ms_per_step_double"]
    return out


def drop_in(reps):
    import pypatchworkpp as m
    fr = kitti()
    objs = {}
    for name in MODES:
        o = m.patchworkpp(m.Parameters())
        o.setArithmetic(name)
        objs[name] = o

    def one(o):
        for a in fr:
            o.estimateGround(a)
            o.getGroundIndices(); o.getNongroundIndices()
    for o in objs.values():
        for _ in range(3):
            one(o)
    times = {k: [] for k in objs}
    for _ in range(reps):
        for name, o in objs.items():
            t0 = time.perf_counter(); one(o); times[name].append((time.perf_counter() - t0) / len(fr) * 1e3)
    out = {"record": "drop_in", "frames": "six recorded KITTI scans, one per call", "rounds": reps}
    for name in objs:
        out[f"ms_per_frame_{name}"] = float(np.median(times[name]))
        out[f"ms_per_frame_{name}_runs"] = times[name]
    import pwpp_b200   # the stage times of one profiled one-frame call per mode (largest patch of the scan: its fit is the tail)
    for name, mode in MODES.items():
        e = pwpp_b200.Engine(device=0)
        e.set_arithmetic(mode)
        e.estimate_host([fr[0]])
        e.set_profiling(True)
        e.estimate_host([fr[0]])
        out[f"stage_ms_{name}"] = e.stage_times_ms()
        if name == "reference":
            out["largest_patch_points"] = max(r.n for r in e.bin_results(0))
        e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    recs = [gpu_info(), batch("synthetic", a.steps, a.reps), batch("kitti_cycled", a.steps, a.reps), drop_in(4 * a.reps)]
    lines = [json.dumps(r) for r in recs]
    print("\n".join(lines))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
