"""What per-frame actions of bound calls cost (pwpp_bind_call_actions). One JSON line per record on stdout and in --out. Run on the
GPU from the repository root after build():

  python tools/bound_actions_bench.py [--parent DIR] [--out FILE]

  gpu       card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  one_frame one KITTI frame (kitti_000000 as 16-byte records on the device, its count in a device tensor): a CUDA-graph replay of
            the call bound with all-RUN actions against the same call bound without actions. Host wall time of one replay ending
            in a stream synchronise, and device time between CUDA events around it; median of --reps replays, three alternated
            runs whose order inside a run flips each time; every record carries the SM clock sampled during its window
  ragged    64 KITTI-shaped sensors (the six fixture scans cycled, 16-byte records) with a fixed seeded schedule that drops 10 % of
            the frames: a CUDA-graph replay of the call bound with actions (SKIP for the dropped frames), against today's only
            exact alternative without actions: read the counts and the schedule back, build the present frames' stream table on
            the host and call pwpp_estimate_device_records on them. Both write the step's schedule into the device tensor first
            (a device-to-device copy from a precomputed table). Medians of --reps steps, three alternated runs, order flipped as
            above, SM clock in every record
  bench     bench.py --gpus 1 --steps 10 --warmup 3 of this tree and of the parent tree --parent (built completely, its oracle
            binaries included: a bench line that reports an error stops the run), alternated
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
for p in (os.path.join(REPO, "tools"), PKG, os.path.join(PKG, "lib"), REPO):
    if p not in sys.path:
        sys.path.insert(0, p)

from bound_call_bench import emit, layout16, timed  # noqa: E402

SEED = 20261017


def timed_with_clocks(fn, reps, stream):
    """timed() plus the SM clock and clock-event reasons sampled while it runs (bench.py's samplers: NVML every 5 ms inside the
    window, the nvidia-smi 200 ms loop as the fallback)."""
    import bench
    smi, nvml = bench.ClockSampler(0), bench.NvmlSampler(0)
    smi.start(); nvml.start()
    t0 = time.perf_counter()
    h, d = timed(fn, reps, stream)
    t1 = time.perf_counter()
    clk_smi = smi.stop()
    clk = nvml.stop(t0, t1)
    if clk is None:
        clk = dict(clk_smi, source="nvidia-smi, 200 ms period")
    return h, d, clk


def rounds(names):
    """Three alternated runs; the order of the paths inside a run flips from one run to the next, so no path always goes first."""
    for rnd in range(3):
        yield rnd, (names if rnd % 2 == 0 else names[::-1])


def scan(k):
    z = np.load(os.path.join(REPO, "tests", "golden", f"kitti_{k:06d}.npz"))
    return np.ascontiguousarray(z["xyzi_t"].T, dtype=np.float32)


def one_frame_leg(args, out):
    import torch
    import pwpp_b200
    s = torch.from_numpy(scan(0)).cuda()
    n = s.shape[0]
    rec = s.view(torch.uint8).reshape(-1).clone()
    counts = torch.tensor([n], dtype=torch.int64, device="cuda")
    actions = torch.zeros(1, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    lay = layout16()
    plain, act = pwpp_b200.Engine(device=0), pwpp_b200.Engine(device=0)
    plain.bind_call([rec.data_ptr()], [n], [lay], counts)
    act.bind_call([rec.data_ptr()], [n], [lay], counts, actions=actions)
    graphs = {}
    with torch.cuda.stream(st):
        for name, e in (("bound_without_actions", plain), ("bound_all_run_actions", act)):
            for _ in range(3):
                e.run_bound_call(st.cuda_stream)
            st.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                e.run_bound_call(torch.cuda.current_stream().cuda_stream)
            graphs[name] = g
    torch.cuda.synchronize()

    def replay(g):
        def fn():
            with torch.cuda.stream(st):
                g.replay()
        return fn

    for g in graphs.values():
        for _ in range(20):
            replay(g)()
    st.synchronize()
    for rnd, names in rounds(list(graphs)):
        for name in names:
            h, d, clk = timed_with_clocks(replay(graphs[name]), args.reps, st)
            emit({"record": "one_frame", "path": name, "run": rnd, "points": n, "host_us_median": round(h, 1), "device_us_median": round(d, 1),
                  "reps": args.reps, "clocks": clk}, out)
    plain.close(); act.close()


def ragged_leg(args, out):
    import torch
    import pwpp_b200
    F = 64
    scans = [scan(k) for k in range(6)]
    data = [torch.from_numpy(scans[f % 6]).cuda().view(torch.uint8).reshape(-1).clone() for f in range(F)]
    sizes = [len(scans[f % 6]) for f in range(F)]
    ptrs = [d.data_ptr() for d in data]
    lay = layout16()
    counts = torch.tensor(sizes, dtype=torch.int64, device="cuda")
    rng = np.random.default_rng(SEED)
    K = 32   # schedules cycled through the timed steps
    table = np.where(rng.random((K, F)) < 0.10, pwpp_b200.FRAME_SKIP, pwpp_b200.FRAME_RUN).astype(np.int32)
    sched = torch.from_numpy(table).cuda()
    actions = torch.zeros(F, dtype=torch.int32, device="cuda")
    h_counts = torch.empty(F, dtype=torch.int64, pin_memory=True)
    h_actions = torch.empty(F, dtype=torch.int32, pin_memory=True)
    st = torch.cuda.Stream()
    bound, direct = pwpp_b200.Engine(device=0, num_streams=F), pwpp_b200.Engine(device=0, num_streams=F)
    bound.bind_call(ptrs, sizes, [lay] * F, counts, actions=actions)
    with torch.cuda.stream(st):
        for _ in range(3):
            bound.run_bound_call(st.cuda_stream)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            bound.run_bound_call(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    step = {"k": 0}

    def graph_step():
        k = step["k"] = (step["k"] + 1) % K
        with torch.cuda.stream(st):
            actions.copy_(sched[k], non_blocking=True)
            g.replay()

    def direct_step():
        k = step["k"] = (step["k"] + 1) % K
        with torch.cuda.stream(st):
            actions.copy_(sched[k], non_blocking=True)
            h_counts.copy_(counts, non_blocking=True)
            h_actions.copy_(actions, non_blocking=True)
        st.synchronize()   # the host needs the counts and the schedule
        c, a = h_counts.numpy(), h_actions.numpy()
        present = [f for f in range(F) if a[f] == pwpp_b200.FRAME_RUN]
        direct.estimate_device_records([ptrs[f] for f in present], [int(c[f]) for f in present], [lay] * len(present), streams=present,
                                       stream=st.cuda_stream)

    legs = {"graph_replay_with_actions": graph_step, "count_read_and_present_frames_call": direct_step}
    for fn in legs.values():
        for _ in range(K):
            fn()
    st.synchronize()
    for rnd, names in rounds(list(legs)):
        for name in names:
            h, d, clk = timed_with_clocks(legs[name], args.ragged_reps, st)
            emit({"record": "ragged", "path": name, "run": rnd, "frames": F, "drop": 0.10, "seed": SEED, "schedules": K,
                  "present_frames_mean": float((table == 0).sum(1).mean()), "host_us_median": round(h, 1), "device_us_median": round(d, 1),
                  "reps": args.ragged_reps, "clocks": clk}, out)
    bound.close(); direct.close()


def bench_legs(args, out):
    trees = [("this", REPO)] + ([("parent", os.path.abspath(args.parent))] if args.parent else [])
    for rnd in range(args.bench_runs):
        for tag, tree in trees:
            res = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", "10", "--warmup", "3"], capture_output=True,
                                 text=True, cwd=tree, timeout=3600)
            assert res.returncode == 0, res.stderr[-2000:]
            line = json.loads([l for l in res.stdout.splitlines() if l.startswith("{")][-1])
            bad = [k for k, v in line.items() if isinstance(v, dict) and "error" in v]
            assert not bad, f"bench.py of the {tag} tree reported errors in {bad}: build that tree completely (its oracle included)"
            emit({"record": "bench", "tree": tag, "run": rnd, "line": line}, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--parent", default="", help="the parent commit's tree, built, for the bench.py A/B")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--ragged-reps", type=int, default=100)
    ap.add_argument("--bench-runs", type=int, default=2)
    ap.add_argument("--legs", default="one_frame,ragged,bench")
    args = ap.parse_args()
    import stream_map_bench
    emit(stream_map_bench.gpu_info(), args.out)
    legs = args.legs.split(",")
    if "one_frame" in legs:
        one_frame_leg(args, args.out)
    if "ragged" in legs:
        ragged_leg(args, args.out)
    if "bench" in legs:
        bench_legs(args, args.out)
    emit(stream_map_bench.gpu_info(), args.out)


if __name__ == "__main__":
    main()
