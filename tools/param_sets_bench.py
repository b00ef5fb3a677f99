"""What several parameter sets in one context (pwpp_create_sets) buy, and what they cost the calls that do not use them. One JSON
line per record on stdout and in --out. Run on the GPU from the repository root after build():

  python tools/param_sets_bench.py [--parent PKG] [--out FILE]

  gpu        card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  ab         bench.py's default workload (1024 synthetic KITTI-64 frames resident in HBM, one pwpp_estimate_device call per step),
             its `streaming` record (64 streams x 16 calls, state carried) and the one-frame latency of estimateGround plus both
             index getters on the recorded scan kitti_000000 (host input, median of 300 calls), with the package directory named
             by --parent (the parent commit's patchwork-plusplus_b200/ with its built lib/) and with this tree's, alternated,
             three runs each, every run in a fresh process
  fleet      48 sensors, 16 ticks of device-resident synthetic KITTI-64 scans: 16 sensors on each of the `default`, `ros` and
             `no_rvpf_tgr` sets of tests/param_sets.py. One context with three sets (one call per tick), three one-set contexts
             (three calls per tick) and one context per sensor (48 one-frame calls per tick)
  eight_sets 8 sensors with 8 different sensor_height / min_range / max_range settings, 16 ticks: one context with eight sets
             against eight one-set contexts
Times are CUDA-event times of a whole pass (all ticks), median of --reps passes; every pass starts from the constructor state.
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
for p in (os.path.join(REPO, "tools"), PKG, os.path.join(PKG, "lib"), REPO, os.path.join(REPO, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def one_frame_latency(pwpp_b200, reps=300):
    z = np.load(os.path.join(REPO, "tests", "golden", "kitti_000000.npz"))
    a = np.ascontiguousarray(z["xyzi_t"].T, dtype=np.float32)
    eng = pwpp_b200.Engine(device=0, num_streams=1)
    for _ in range(20):
        eng.estimate_host([a]); eng.ground_indices(0); eng.nonground_indices(0)
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        eng.estimate_host([a]); eng.ground_indices(0); eng.nonground_indices(0)
        t.append(time.perf_counter() - t0)
    eng.close()
    return {"one_frame_us_median": float(np.median(t)) * 1e6, "one_frame_us_p10": float(np.percentile(t, 10)) * 1e6}


def ab_child(pkg, steps, warmup):
    sys.path.insert(0, pkg)
    import stream_map_bench
    import pwpp_b200
    r = stream_map_bench.ab_leg(pkg, steps, warmup)
    r.update(one_frame_latency(pwpp_b200))
    return r


def gpu_info():
    import stream_map_bench
    return stream_map_bench.gpu_info()


def ticks_device(sets_of_sensor, ticks, seed):
    """Per tick: the scans of all sensors back to back on the device (sensor order), and their offsets."""
    import synth
    import torch
    dev = torch.device("cuda", 0)
    S = len(sets_of_sensor)
    out = []
    for t in range(ticks):
        pts, offs = synth.make_batch(seed, t * S, S, "kitti64", dev)
        out.append((pts.contiguous(), offs.numpy().astype(np.int64)))
    torch.cuda.synchronize()
    return out


def timed(fn, reps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn(); torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms


def fleet_record(sets, sensor_set, ticks, reps, seed, groups):
    """One context with every set, one context per set (`groups` = True) and one context per sensor, on the same ticks. The
    contexts of each setup exist only while it is timed."""
    import pwpp_b200
    import torch
    S = len(sensor_set)
    data = ticks_device(sensor_set, ticks, seed)
    stream = torch.cuda.current_stream().cuda_stream
    maxn = int(max(np.diff(o).max() for _, o in data))
    res = {"sensors": S, "ticks": ticks, "frames": S * ticks, "reps": reps}

    def setup_multi():
        e = pwpp_b200.Engine(sets, device=0, num_streams=S, max_points_per_frame=maxn, stream_set=sensor_set)
        calls = [(e, 0, S)]
        return [e], calls

    def setup_groups():
        engs, calls = [], []
        for k in range(len(sets)):
            members = [s for s in range(S) if sensor_set[s] == k]
            assert members == list(range(members[0], members[0] + len(members))), "the sensors of a set are consecutive"
            e = pwpp_b200.Engine(sets[k], device=0, num_streams=len(members), max_points_per_frame=maxn)
            engs.append(e); calls.append((e, members[0], len(members)))
        return engs, calls

    def setup_sensors():
        engs = [pwpp_b200.Engine(sets[sensor_set[s]], device=0, num_streams=1, max_points_per_frame=maxn) for s in range(S)]
        return engs, [(e, s, 1) for s, e in enumerate(engs)]

    heights = {}
    for name, setup in (("one_context_all_sets", setup_multi), ("one_context_per_set", setup_groups if groups else None),
                        ("one_context_per_sensor", setup_sensors)):
        if setup is None:
            continue
        print(f"[param_sets_bench] {name}: {S} sensors, {ticks} ticks", file=sys.stderr, flush=True)
        engs, calls = setup()

        def run():
            for e in engs:
                e.reset()
            for pts, offs in data:
                for e, first, cnt in calls:
                    e.estimate_device(pts.data_ptr() + int(offs[first]) * 16, offs[first:first + cnt + 1] - offs[first], True, stream)
        ms = timed(run, reps)
        res[name] = {"ms_per_pass_median": float(np.median(ms)), "frames_per_s": S * ticks / (float(np.median(ms)) / 1e3), "ms_per_pass_runs": ms}
        heights[name] = [e.height(s - first) for e, first, cnt in calls for s in range(first, first + cnt)]
        for e in engs:
            e.close()
    # the schedules compute the same thing per sensor: the batched ones with the same kernels (bit for bit), one-frame calls with
    # the small-call kernels (planes agree to ~1e-9): the largest difference of the adaptive heights after the last tick
    h0 = np.array(heights["one_context_all_sets"])
    for name in heights:
        if name != "one_context_all_sets":
            res["max_height_diff_vs_" + name] = float(np.abs(np.array(heights[name]) - h0).max())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default="", help="patchwork-plusplus_b200/ directory of the parent build for the A/B leg ('' = skip it)")
    ap.add_argument("--out", default="")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--leg", default="", help=argparse.SUPPRESS)
    ap.add_argument("--pkg", default=PKG, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.leg == "ab":
        print(json.dumps(ab_child(args.pkg, args.steps, args.warmup)), flush=True)
        return
    records = [gpu_info()]
    print(json.dumps(records[0]), flush=True)
    emit = lambda r: (records.append(r), print(json.dumps(r), flush=True))   # noqa: E731
    if args.parent:
        for rep in range(3):
            for tag, pkg in (("parent", os.path.abspath(args.parent)), ("this", PKG)):
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--leg", "ab", "--pkg", pkg, "--steps", str(args.steps),
                                      "--warmup", str(args.warmup)], capture_output=True, text=True, cwd=REPO, timeout=900)
                if out.returncode != 0:
                    raise RuntimeError(out.stderr[-2000:])
                emit({"record": "ab", "build": tag, "run": rep, "steps": args.steps, **json.loads(out.stdout.strip().splitlines()[-1])})
    from param_sets import PARAM_SETS
    import bench
    sets = [PARAM_SETS[n][0]() for n in ("default", "ros", "no_rvpf_tgr")]
    emit({"record": "fleet", "sets": ["default", "ros", "no_rvpf_tgr"], "sensors_per_set": 16,
          **fleet_record(sets, [k for k in range(3) for _ in range(16)], 16, args.reps, bench.SEED, True)})
    eight = []
    for k in range(8):
        p = PARAM_SETS["default"][0]()
        p.sensor_height = 1.5 + 0.1 * k
        p.min_range = 2.0 + 0.25 * k
        p.max_range = 60.0 + 5.0 * k
        eight.append(p)
    emit({"record": "eight_sets", "sensor_height": [round(p.sensor_height, 3) for p in eight], "min_range": [p.min_range for p in eight],
          "max_range": [p.max_range for p in eight], **fleet_record(eight, list(range(8)), 16, args.reps, bench.SEED + 1, False)})
    if args.out:
        with open(args.out, "w") as fh:
            for r in records:
                fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
