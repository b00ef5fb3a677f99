"""What bound calls cost and save (pwpp_bind_call / pwpp_run_bound_call). One JSON line per record on stdout and in --out. Run on
the GPU from the repository root after build():

  python tools/bound_call_bench.py [--parent DIR] [--out FILE]

  gpu       card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  latency   one KITTI frame (kitti_000000 as 16-byte records on the device, its count in a device tensor): a CUDA-graph replay of
            the bound call against pwpp_estimate_device_records preceded by a device-to-host read of the count, both on one
            stream. Host wall time of one call ending in a stream synchronise, and device time between CUDA events around it;
            median of --reps calls, three alternating runs
  batch     bench.py's 1024-frame KITTI-64 batch as 16-byte records: an eager run of the bound call (capacities = the frame
            sizes, and 1.5 x the largest frame for every frame), pwpp_estimate_device_records with host sizes, and
            pwpp_estimate_device on the pre-packed float4 batch (no unpack). Device time between CUDA events, median of --reps
            calls, three alternating runs
  bench     bench.py --gpus 1 --steps 10 --warmup 3 of this tree and of the parent tree --parent (built), alternated
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
for p in (os.path.join(REPO, "tools"), PKG, os.path.join(PKG, "lib"), REPO):
    if p not in sys.path:
        sys.path.insert(0, p)


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def layout16():
    import pwpp_b200
    L = pwpp_b200.PwppPointLayout()
    L.point_step = 16
    L.offset[:] = [0, 4, 8, 12]
    L.datatype[:] = [7, 7, 7, 7]
    return L


def timed(fn, reps, stream):
    """(host wall us, device us) medians of fn() over reps calls, each ending in a synchronise of stream."""
    import torch
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    host, dev = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        ev0.record(stream)
        fn()
        ev1.record(stream)
        stream.synchronize()
        host.append((time.perf_counter() - t0) * 1e6)
        dev.append(ev0.elapsed_time(ev1) * 1e3)
    return float(np.median(host)), float(np.median(dev))


def latency_leg(args, out):
    import torch
    import pwpp_b200
    z = np.load(os.path.join(REPO, "tests", "golden", "kitti_000000.npz"))
    scan = torch.from_numpy(np.ascontiguousarray(z["xyzi_t"].T, dtype=np.float32)).cuda()
    n = scan.shape[0]
    rec = scan.view(torch.uint8).reshape(-1).clone()   # 16-byte records: the float4 layout
    counts = torch.tensor([n], dtype=torch.int64, device="cuda")
    st = torch.cuda.Stream()
    lay = layout16()
    bound, direct = pwpp_b200.Engine(device=0), pwpp_b200.Engine(device=0)
    bound.bind_call([rec.data_ptr()], [n], [lay], counts)
    with torch.cuda.stream(st):
        for _ in range(3):
            bound.run_bound_call(st.cuda_stream)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            bound.run_bound_call(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()

    def replay():
        with torch.cuda.stream(st):
            g.replay()

    def records_call():
        k = int(counts.item())   # the count read back to the host
        direct.estimate_device_records([rec.data_ptr()], [k], [lay], stream=st.cuda_stream)

    for _ in range(20):
        replay(); records_call()
    st.synchronize()
    for rnd in range(3):
        for name, fn in (("graph_replay", replay), ("device_records_after_count_read", records_call)):
            h, d = timed(fn, args.reps, st)
            emit({"record": "latency", "path": name, "run": rnd, "points": n, "host_us_median": round(h, 1), "device_us_median": round(d, 1),
                  "reps": args.reps}, out)
    bound.close(); direct.close()


def batch_leg(args, out):
    import torch
    import bench
    import pwpp_b200
    import synth
    F = 1024
    pts, offs = synth.make_batch(bench.SEED, 0, F, "kitti64", torch.device("cuda", 0))
    offs_np = offs.numpy().astype(np.int64)
    sizes = np.diff(offs_np)
    lay = layout16()
    rec = pts.view(torch.uint8).reshape(-1)
    ptrs = [rec.data_ptr() + int(o) * 16 for o in offs_np[:-1]]
    counts = torch.from_numpy(sizes.copy()).cuda()
    st = torch.cuda.Stream()
    cap_pad = int(sizes.max() * 3 // 2)
    eng = pwpp_b200.Engine(device=0, num_streams=F)
    pad = pwpp_b200.Engine(device=0, num_streams=F)
    eng.bind_call(ptrs, sizes.tolist(), [lay] * F, counts)     # direct calls of the same sizes fit its frozen buffers
    # every frame's capacity 1.5 x the largest frame: frame f's capacity runs into frame f + 1's records, which are never
    # read past the count; the buffer ends one capacity after the last frame's start
    big = torch.zeros(int(offs_np[-1] + cap_pad) * 16, dtype=torch.uint8, device="cuda")
    big[: rec.numel()] = rec
    pad.bind_call([big.data_ptr() + int(o) * 16 for o in offs_np[:-1]], [cap_pad] * F, [lay] * F, counts)
    torch.cuda.synchronize()
    offs_c = (C.c_int64 * (F + 1))(*offs_np.tolist())

    legs = {
        "bound_call_capacity_equals_size": lambda: eng.run_bound_call(st.cuda_stream),
        "bound_call_capacity_1.5x_largest": lambda: pad.run_bound_call(st.cuda_stream),
        "device_records_host_sizes": lambda: eng.estimate_device_records(ptrs, sizes.tolist(), [lay] * F, stream=st.cuda_stream),
        "device_packed_float4": lambda: eng.lib.pwpp_estimate_device(eng._h, F, C.c_void_p(pts.data_ptr()), offs_c, 1, C.c_void_p(st.cuda_stream)),
    }
    for fn in legs.values():
        for _ in range(2):
            fn()
    st.synchronize()
    for rnd in range(3):
        for name, fn in legs.items():
            h, d = timed(fn, args.batch_reps, st)
            emit({"record": "batch", "path": name, "run": rnd, "frames": F, "points": int(offs_np[-1]), "host_us_median": round(h, 1),
                  "device_us_median": round(d, 1), "reps": args.batch_reps}, out)
    eng.close(); pad.close()


def bench_legs(args, out):
    trees = [("this", REPO)] + ([("parent", os.path.abspath(args.parent))] if args.parent else [])
    for rnd in range(args.bench_runs):
        for tag, tree in trees:
            res = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", "10", "--warmup", "3"], capture_output=True,
                                 text=True, cwd=tree, timeout=3600)
            assert res.returncode == 0, res.stderr[-2000:]
            line = [l for l in res.stdout.splitlines() if l.startswith("{")][-1]
            emit({"record": "bench", "tree": tag, "run": rnd, "line": json.loads(line)}, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--parent", default="", help="the parent commit's tree, built, for the bench.py A/B")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--batch-reps", type=int, default=30)
    ap.add_argument("--bench-runs", type=int, default=1)
    ap.add_argument("--legs", default="latency,batch,bench")
    args = ap.parse_args()
    import stream_map_bench
    emit(stream_map_bench.gpu_info(), args.out)
    legs = args.legs.split(",")
    if "latency" in legs:
        latency_leg(args, args.out)
    if "batch" in legs:
        batch_leg(args, args.out)
    if "bench" in legs:
        bench_legs(args, args.out)
    emit(stream_map_bench.gpu_info(), args.out)


if __name__ == "__main__":
    main()
