"""What the stream table (pwpp_estimate_host_streams) buys, and what it costs the calls that do not use it. One JSON line per
record on stdout and in --out. Run on the GPU from the repository root after build():

  python tools/stream_map_bench.py [--parent PKG] [--out FILE]

  gpu        card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  ab         bench.py's default workload (1024 synthetic KITTI-64 frames resident in HBM, every frame on a fresh stream, one
             pwpp_estimate_device call per step) and its `streaming` record (64 streams x 16 calls, state carried), with the
             package directory named by --parent (the parent commit's patchwork-plusplus_b200/ with its built lib/) and with
             this tree's, alternated, three runs each, every run in a fresh process
  one_stream 64 recorded KITTI scans of ONE stream from page-locked memory: 64 one-frame calls, 8 calls of 8 frames, one call
             of 64 frames (wall clock per pass, end to end: upload, kernels, index lists back on the host)
  ragged     64 sensors with 4..12 scans each and ~10 % of the scans dropped, delivered tick by tick: one call per tick naming
             the sensors that have a scan (pwpp_estimate_host_streams), against one context per sensor and one-frame calls
"""
import argparse
import ctypes as C
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


def gpu_info():
    q = "name,power.limit,clocks.max.sm,driver_version"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, clk, drv = [x.strip() for x in out[0].split(",")]
    return {"record": "gpu", "name": name, "power_limit": plim, "max_sm_clock": clk, "driver": drv}


def ab_leg(pkg, steps, warmup):
    """bench.py's default step and streaming record, with the package (wrapper + library) in directory pkg."""
    sys.path.insert(0, pkg)
    import torch
    import bench
    import pwpp_b200
    import synth
    F = 1024
    dev = torch.device("cuda", 0)
    pts, offs = synth.make_batch(bench.SEED, 0, F, "kitti64", dev)
    offs_np = offs.numpy()
    eng = pwpp_b200.Engine(device=0, num_streams=F, max_points_per_frame=int(np.diff(offs_np).max()))
    ts = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(ts)
    stream = ts.cuda_stream

    def step():
        eng.reset()
        eng.estimate_device(pts.data_ptr(), offs_np, True, stream)
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record(); torch.cuda.synchronize()
    ms_step = e0.elapsed_time(e1) / steps
    eng.close()
    S, T = 64, 16
    seng = pwpp_b200.Engine(device=0, num_streams=S, max_points_per_frame=int(np.diff(offs_np).max()))
    calls = [(int(offs_np[t * S]), (offs_np[t * S:(t + 1) * S + 1] - offs_np[t * S]).copy()) for t in range(T)]

    def sequence():
        seng.reset()
        for first, o in calls:
            seng.estimate_device(pts.data_ptr() + first * 16, o, True, stream)
    sequence(); torch.cuda.synchronize()
    e0.record()
    for _ in range(3):
        sequence()
    e1.record(); torch.cuda.synchronize()
    ms_seq = e0.elapsed_time(e1) / 3
    seng.close()
    return {"ms_per_step": ms_step, "frames_per_s": F / (ms_step / 1e3), "streaming_ms_per_sequence": ms_seq, "streaming_frames_per_s": S * T / (ms_seq / 1e3)}


class Pinned:
    """The six recorded KITTI scans (tests/golden/) in page-locked memory allocated by the library."""

    def __init__(self, lib):
        self.lib, self.ptrs, self.arrays = lib, [], []
        for k in range(6):
            z = np.load(os.path.join(REPO, "tests", "golden", f"kitti_{k:06d}.npz"))
            a = np.ascontiguousarray(z["xyzi_t"].T, dtype=np.float32)
            p = lib.pwpp_host_alloc(a.nbytes)
            v = np.ctypeslib.as_array((C.c_float * a.size).from_address(p)).reshape(a.shape)
            v[:] = a
            self.ptrs.append(p); self.arrays.append(v)

    def free(self):
        for p in self.ptrs:
            self.lib.pwpp_host_free(p)


def one_stream(pinned, reps):
    import pwpp_b200
    frames = [pinned.arrays[t % 6] for t in range(64)]
    eng = pwpp_b200.Engine(device=0, num_streams=1)
    out = {}
    for k in (1, 8, 64):
        def one_pass():
            eng.reset()
            for c in range(0, 64, k):
                eng.estimate_host(frames[c:c + k], streams=[0] * k)
        one_pass()
        times = []
        for _ in range(reps):
            t0 = time.perf_counter(); one_pass(); times.append(time.perf_counter() - t0)
        out[f"frames_per_call_{k}"] = {"calls": 64 // k, "s_per_pass_median": float(np.median(times)), "frames_per_s": 64 / float(np.median(times)),
                                      "frames_per_s_runs": [64 / t for t in times]}
    eng.close()
    return out


def ragged(pinned, reps):
    import pwpp_b200
    rng = np.random.default_rng(7)
    S = 64
    lengths = rng.integers(4, 13, S)
    ticks = []   # per tick: the sensors that deliver a scan (dropped scans never arrive)
    for t in range(int(lengths.max())):
        ticks.append([s for s in range(S) if t < lengths[s] and rng.random() >= 0.1])
    nframes = sum(len(x) for x in ticks)
    scan = lambda s, t: pinned.arrays[(s + t) % 6]   # noqa: E731
    eng = pwpp_b200.Engine(device=0, num_streams=S)

    def batched():
        eng.reset()
        for t, ss in enumerate(ticks):
            if ss:
                eng.estimate_host([scan(s, t) for s in ss], streams=ss)
    per = [pwpp_b200.Engine(device=0, num_streams=1) for _ in range(S)]

    def per_sensor():
        for e in per:
            e.reset()
        for t, ss in enumerate(ticks):
            for s in ss:
                per[s].estimate_host([scan(s, t)])
    res = {"streams": S, "frames": nframes, "ticks": len(ticks), "scans_per_stream": [int(x) for x in lengths],
           "dropped": int(lengths.sum()) - nframes}
    for name, fn in (("stream_table", batched), ("context_per_sensor", per_sensor)):
        fn()
        times = []
        for _ in range(reps):
            t0 = time.perf_counter(); fn(); times.append(time.perf_counter() - t0)
        res[name] = {"s_per_pass_median": float(np.median(times)), "frames_per_s": nframes / float(np.median(times)),
                     "frames_per_s_runs": [nframes / t for t in times]}
    # the two schedules compute the same thing (batched calls take the batch kernels, one-frame calls the small-call kernels:
    # planes agree to ~1e-9, not bit for bit)
    for s in range(S):
        assert abs(eng.height(s) - per[s].height(0)) <= 1e-9, f"sensor {s}: adaptive height differs between the two schedules"
    for e in per:
        e.close()
    eng.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default="", help="patchwork-plusplus_b200/ directory of the parent build for the A/B leg ('' = skip it)")
    ap.add_argument("--out", default="")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--leg", default="", help=argparse.SUPPRESS)   # internal: one A/B run in a child process
    ap.add_argument("--pkg", default=PKG, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.leg == "ab":
        print(json.dumps(ab_leg(args.pkg, args.steps, args.warmup)), flush=True)
        return
    records = [gpu_info()]
    emit = lambda r: (records.append(r), print(json.dumps(r), flush=True))   # noqa: E731
    print(json.dumps(records[0]), flush=True)
    if args.parent:
        for rep in range(3):
            for tag, pkg in (("parent", os.path.abspath(args.parent)), ("this", PKG)):
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--leg", "ab", "--pkg", pkg, "--steps", str(args.steps),
                                      "--warmup", str(args.warmup)], capture_output=True, text=True, cwd=REPO, timeout=900)
                if out.returncode != 0:
                    raise RuntimeError(out.stderr[-2000:])
                emit({"record": "ab", "build": tag, "run": rep, "steps": args.steps, **json.loads(out.stdout.strip().splitlines()[-1])})
    import pwpp_b200
    pinned = Pinned(pwpp_b200.load_library())
    try:
        emit({"record": "one_stream", "scans": 64, "source": "tests/golden kitti_00000{0..5} cycled, page-locked", "reps": args.reps, **one_stream(pinned, args.reps)})
        emit({"record": "ragged", "reps": args.reps, **ragged(pinned, args.reps)})
    finally:
        pinned.free()
    if args.out:
        with open(args.out, "w") as fh:
            for r in records:
                fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
