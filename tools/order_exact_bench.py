"""What PWPP_ORDER_REFERENCE_EXACT (the libstdc++ tie order, csrc/pwpp_order_exact.cuh) costs over PWPP_ORDER_REFERENCE, and how
many patches need it. One JSON line per record on stdout and in --out. Run on the GPU from the repository root after build():

  python tools/order_exact_bench.py [--steps K] [--reps R] [--out FILE]

  gpu       card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  batch     step time of one pwpp_estimate_device call over 1024 frames resident in HBM (every frame on a fresh stream), for
            bench.py's synthetic KITTI-64 batch and for the six recorded KITTI scans cycled to 1024 frames; the two orders
            alternate, R rounds of K steps each (CUDA events); with the fix-up's counters per frame (patches simulated, heap
            fall-backs, NaN bins)
  drop_in   one-frame latency of the drop-in class's pattern (estimateGround + both index getters: upload, kernels, lists back on
            the host) over the six recorded scans, both orders alternating, wall clock
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

ORDERS = {"reference": 1, "reference_exact": 2}


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
    for name, order in ORDERS.items():
        e = pwpp_b200.Engine(device=0, num_streams=F, max_points_per_frame=int(np.diff(offs_np).max()))
        e.set_output_order(order)
        engs[name] = e

    def step(e):
        e.reset()
        e.estimate_device(pts.data_ptr(), offs_np, True, ts.cuda_stream)
    out = {"record": "batch", "workload": workload, "frames": F, "points": int(offs_np[-1]), "steps": steps, "rounds": reps}
    for name, e in engs.items():   # warm-up, and the counters of one step
        for _ in range(3):
            step(e)
        torch.cuda.synchronize()
        if name == "reference_exact":
            e.order_exact_counts(reset=True)
            step(e)
            c = e.order_exact_counts()
            out["per_frame"] = {"patches_simulated": c[0] / F, "heap_fallbacks": c[1] / F, "nan_bins": c[2] / F}
            out["patches_per_frame"] = sum(e.num_patches(f) for f in range(F)) / F
        out[f"launches_per_step_{name}"] = None
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
    out["exact_over_reference"] = out["ms_per_step_reference_exact"] / out["ms_per_step_reference"]
    return out


def drop_in(reps):
    import pypatchworkpp as m
    fr = kitti()
    objs = {}
    for name in ORDERS:
        o = m.patchworkpp(m.Parameters())
        o.setOutputOrder(name)
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
