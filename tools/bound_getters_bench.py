"""What the getter results of a bound call cost (pwpp_bind_getter_results: k_gather_xyz_parts, k_bound_states). One JSON line per
record on stdout and in --out. Run on the GPU from the repository root after build():

  python tools/bound_getters_bench.py [--out FILE]

  gpu       card name, power limit, maximum and current SM clock (nvidia-smi), read before and after the numbers in the same command
  latency   one KITTI frame (kitti_000000) as 16-byte records: a CUDA-graph replay of the bound call with nothing enabled, with both
            xyz parts, with the state, and with everything, alternated. Device time between CUDA events around one replay, median
            of --reps replays, three runs
  tick      64 KITTI-64 sensors as 22-byte (velodyne) records, one bound call: (a) a graph replay with every getter result in the
            graph, ended by a device synchronise; (b) a replay without them, a synchronise, then the host getters of every frame
            (pwpp_copy_ground_xyz, pwpp_copy_nonground_xyz, pwpp_copy_centers, pwpp_copy_normals, pwpp_get_state). Host clock
            around each tick, median of --ticks ticks, paths alternated, three runs
  gather    bench.py's 1024-frame KITTI-64 batch as 16-byte records in one bound call with both xyz parts and both record parts
            enabled: k_gather_xyz_parts against k_gather_record_parts on the same lists (kernel times from torch.profiler over
            --kreps runs), next to a device-to-device copy with the xyz gather's HBM traffic (4 + 16 + 12 bytes per listed point;
            a copy of 16 bytes per listed point moves 32), three runs
"""
import argparse
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

import bound_records_bench  # noqa: E402  (batch, kernel_times)
import records_bench  # noqa: E402  (make_records, layout, emit)

emit = records_bench.emit
VARIANTS = {"none": None, "xyz": (True, True, False), "state": (False, False, True), "all": (True, True, True)}


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,driver_version"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, clk, cur, drv = [x.strip() for x in out[0].split(",")]
    return {"record": "gpu", "name": name, "power_limit": plim, "max_sm_clock": clk, "sm_clock": cur, "driver": drv}


def capture(e, st):
    import torch
    with torch.cuda.stream(st):
        for _ in range(3):
            e.run_bound_call(st.cuda_stream)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            e.run_bound_call(torch.cuda.current_stream().cuda_stream)
    return g


def latency_leg(args, out):
    import torch
    import pwpp_b200
    z = np.load(os.path.join(REPO, "tests", "golden", "kitti_000000.npz"))
    pts = torch.from_numpy(np.ascontiguousarray(z["xyzi_t"].T, dtype=np.float32)).cuda()
    n = pts.shape[0]
    st = torch.cuda.Stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rec = records_bench.make_records(pts, 16)
    counts = torch.tensor([n], dtype=torch.int64, device="cuda")
    graphs, engines = {}, []
    for variant, what in VARIANTS.items():
        e = pwpp_b200.Engine(device=0)
        e.bind_call([rec.data_ptr()], [n], [records_bench.layout(16)], counts)
        if what:
            e.bind_getter_results(*what)
        graphs[variant] = capture(e, st)
        engines.append(e)
    torch.cuda.synchronize()
    for rnd in range(3):
        for variant, g in graphs.items():
            dev = []
            with torch.cuda.stream(st):
                for _ in range(10):
                    g.replay()
                for _ in range(args.reps):
                    ev0.record(st)
                    g.replay()
                    ev1.record(st)
                    ev1.synchronize()
                    dev.append(ev0.elapsed_time(ev1) * 1e3)
            emit({"record": "latency", "variant": variant, "run": rnd, "points": n, "device_us_median": round(float(np.median(dev)), 1),
                  "reps": args.reps}, out)
    for e in engines:
        e.close()


def tick_leg(args, out, pts, offs_np):
    import torch
    import pwpp_b200
    F = 64
    sizes = np.diff(offs_np)[:F]
    step = 22
    rec = records_bench.make_records(pts[: int(offs_np[F])], step)
    ptrs = [rec.data_ptr() + int(o) * step for o in offs_np[:F]]
    counts = torch.from_numpy(sizes.copy()).cuda()
    lay = records_bench.layout(step)
    st = torch.cuda.Stream()
    paths = {}
    for path in ("graph_getters", "replay_then_host_getters"):
        e = pwpp_b200.Engine(device=0, num_streams=F)
        e.bind_call(ptrs, sizes.tolist(), [lay] * F, counts)
        if path == "graph_getters":
            e.bind_getter_results()
        paths[path] = (e, capture(e, st))
    bufs = [np.empty((int(k), 3), np.float32) for k in sizes]

    def tick(path):
        e, g = paths[path]
        with torch.cuda.stream(st):
            g.replay()
        st.synchronize()
        if path == "replay_then_host_getters":
            e.bound_call_results()   # the host getters now serve the replay
            for f in range(F):
                e.lib.pwpp_copy_ground_xyz(e._h, f, bufs[f].ctypes.data)
                e.lib.pwpp_copy_nonground_xyz(e._h, f, bufs[f].ctypes.data)
                e.centers(f)
                e.normals(f)
                e.state(f)
    for path in paths:
        for _ in range(5):
            tick(path)
    for rnd in range(3):
        for path in (paths if rnd % 2 == 0 else list(paths)[::-1]):
            ts = []
            for _ in range(args.ticks):
                t0 = time.perf_counter()
                tick(path)
                ts.append((time.perf_counter() - t0) * 1e6)
            emit({"record": "tick", "path": path, "run": rnd, "sensors": F, "step": step, "points": int(sizes.sum()),
                  "tick_us_median": round(float(np.median(ts)), 1), "ticks": args.ticks}, out)
    for e, _ in paths.values():
        e.close()


def gather_leg(args, out, pts, offs_np):
    import torch
    import pwpp_b200
    F = len(offs_np) - 1
    sizes = np.diff(offs_np)
    npts = int(offs_np[-1])
    rec = records_bench.make_records(pts, 16)
    ptrs = [rec.data_ptr() + int(o) * 16 for o in offs_np[:-1]]
    e = pwpp_b200.Engine(device=0, num_streams=F)
    e.bind_call(ptrs, sizes.tolist(), [records_bench.layout(16)] * F, torch.from_numpy(sizes.copy()).cuda())
    e.bind_getter_results(state=False)
    e.bind_record_results()
    for _ in range(2):
        e.run_bound_call()
    e.synchronize()
    G = e.bound_getter_results()
    idx, poff, nground, _ = e.bound_call_results()
    for f in (0, F // 2, F - 1):   # the output of the last run against the lists
        o, g, k = int(poff[f]), int(nground[f]), int(G["xyz_counts"][f, 1])
        want = pts[o: o + int(sizes[f])][idx[o + g: o + g + k].long(), :3]
        assert torch.equal(G["nonground_xyz"][int(G["row_off"][f]):][:k].view(torch.int32), want.contiguous().view(torch.int32)), f"frame {f}"
    listed = int(G["xyz_counts"].sum())
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    src = torch.empty(listed * 16, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    dst.copy_(src)
    times = {"k_gather_xyz_parts": [], "k_gather_record_parts": []}
    copy = []
    for rnd in range(3):
        for name in (times if rnd % 2 == 0 else list(times)[::-1]):
            times[name] += bound_records_bench.kernel_times(e.run_bound_call, args.kreps, name, e.synchronize)
        for _ in range(args.kreps):
            ev0.record(); dst.copy_(src); ev1.record(); ev1.synchronize()
            copy.append(ev0.elapsed_time(ev1) * 1e3)
    traffic = {"k_gather_xyz_parts": listed * 32, "k_gather_record_parts": listed * 36}
    cu = float(np.median(copy))
    for name, ts in times.items():
        ku = float(np.median(ts))
        emit({"record": "gather", "kernel": name, "frames": F, "points": npts, "listed": listed, "traffic_bytes": traffic[name],
              "kernel_us_median": round(ku, 1), "kernel_us_min": round(float(np.min(ts)), 1), "kernel_us_max": round(float(np.max(ts)), 1),
              "kernel_GBps": round(traffic[name] / ku / 1e3, 1), "memcpy_bytes": listed * 16, "memcpy_us_median": round(cu, 1),
              "samples": len(ts)}, out)
    e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--ticks", type=int, default=50)
    ap.add_argument("--kreps", type=int, default=10)
    ap.add_argument("--legs", default="latency,tick,gather")
    args = ap.parse_args()
    import torch
    emit(gpu_info(), args.out)
    legs = args.legs.split(",")
    if "latency" in legs:
        latency_leg(args, args.out)
    if "tick" in legs or "gather" in legs:
        pts, offs_np = bound_records_bench.batch(torch.device("cuda", 0))
        if "tick" in legs:
            tick_leg(args, args.out, pts, offs_np)
        if "gather" in legs:
            gather_leg(args, args.out, pts, offs_np)
    emit(gpu_info(), args.out)


if __name__ == "__main__":
    main()
