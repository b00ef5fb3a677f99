"""What unpacking sensor records on the GPU costs (pwpp_estimate_host_records / pwpp_estimate_device_records). One JSON line per
record on stdout and in --out. Run on the GPU from the repository root after build():

  python tools/records_bench.py [--parent DIR] [--out FILE]

  gpu      card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  unpack   the unpack kernel alone (k_unpack_records, kernel time from torch.profiler over --reps calls) on bench.py's 1024-frame
           KITTI-64 batch laid out as records of 16, 22, 32 and 48 bytes, next to a device-to-device cudaMemcpyAsync with the same
           HBM traffic (step + 16 bytes per point: a copy of (step + 16) / 2 bytes per point reads and writes that much), timed
           with CUDA events in the same run
  device   step time of that batch through pwpp_estimate_device_records against pwpp_estimate_device on the pre-packed float4
           batch (host clock around the call and a device synchronise, median of --reps steps), alternated
  host     one-frame latency of estimateGround on kitti_000000 laid out as pcl_xyzi32, velodyne22 and rec48 (x, y, z, intensity
           at 16 of a 48-byte point), pageable and page-locked: the records path, the PointCloud2View path with its host gather,
           and an N x 4 array packed in advance (tools/pc2_latency.cpp, built into a temporary directory)
  bench    bench.py --gpus 1 --steps 10 --warmup 3 of this tree and of the parent tree --parent (built), alternated, three runs each
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, "patchwork-plusplus_b200")
for p in (os.path.join(REPO, "tools"), PKG, os.path.join(PKG, "lib"), REPO):
    if p not in sys.path:
        sys.path.insert(0, p)

STEPS = (16, 22, 32, 48)
INTENSITY_AT = {16: 12, 22: 12, 32: 16, 48: 16}


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def make_records(pts, step):
    """(N, step) uint8 records on the device: x, y, z at 0, 4, 8, intensity at INTENSITY_AT[step], the rest filler."""
    import torch
    pb = pts.view(torch.uint8).reshape(-1, 16)
    rec = torch.full((pb.shape[0], step), 0xAB, dtype=torch.uint8, device=pts.device)
    rec[:, 0:12] = pb[:, 0:12]
    oi = INTENSITY_AT[step]
    rec[:, oi:oi + 4] = pb[:, 12:16]
    return rec


def layout(step):
    import pwpp_b200
    L = pwpp_b200.PwppPointLayout()
    L.point_step = step
    L.offset[:] = [0, 4, 8, INTENSITY_AT[step]]
    L.datatype[:] = [7, 7, 7, 7]
    return L


def device_legs(args, out):
    import torch
    import bench
    import pwpp_b200
    import synth
    from torch.profiler import ProfilerActivity, profile
    F = 1024
    dev = torch.device("cuda", 0)
    pts, offs = synth.make_batch(bench.SEED, 0, F, "kitti64", dev)
    offs_np = offs.numpy().astype(np.int64)
    npts = int(offs_np[-1])
    eng = pwpp_b200.Engine(device=0, num_streams=F, max_points_per_frame=int(np.diff(offs_np).max()))
    lib = eng.lib
    ids = (C.c_int32 * F)(*range(F))
    ns = (C.c_int64 * F)(*np.diff(offs_np).tolist())
    offs_c = (C.c_int64 * (F + 1))(*offs_np.tolist())
    recs = {}
    for step in STEPS:
        r = make_records(pts, step)
        recs[step] = (r, (C.c_void_p * F)(*[r.data_ptr() + int(o) * step for o in offs_np[:-1]]), (pwpp_b200.PwppPointLayout * F)(*([layout(step)] * F)))
    torch.cuda.synchronize()

    def call_records(step):
        _, ptrs, lays = recs[step]
        assert lib.pwpp_estimate_device_records(eng._h, F, ids, ptrs, ns, lays, None) == 0, lib.pwpp_last_error()

    def call_packed():
        assert lib.pwpp_estimate_device(eng._h, F, C.c_void_p(pts.data_ptr()), offs_c, 1, None) == 0, lib.pwpp_last_error()

    for step in STEPS:   # warm every shape
        for _ in range(2):
            call_records(step)
        eng.synchronize()
    for _ in range(2):
        call_packed()
    eng.synchronize()
    unpack = {s: [] for s in STEPS}
    copy = {s: [] for s in STEPS}
    steps = {s: [] for s in STEPS}
    packed = []
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for rnd in range(3):   # variants alternate within the run
        for step in STEPS:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    call_records(step)
                eng.synchronize()
            ks = [e for e in prof.events() if "k_unpack_records" in e.name and e.device_type.name == "CUDA"]
            assert len(ks) == args.reps, len(ks)
            unpack[step] += [e.device_time for e in ks]   # microseconds
            nbytes = npts * (step + 16) // 2
            src = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            dst = torch.empty_like(src)
            dst.copy_(src)
            for _ in range(args.reps):
                ev0.record(); dst.copy_(src); ev1.record(); ev1.synchronize()
                copy[step].append(ev0.elapsed_time(ev1) * 1e3)
            del src, dst
            for _ in range(args.reps):
                t0 = time.perf_counter(); call_records(step); eng.synchronize(); steps[step].append((time.perf_counter() - t0) * 1e3)
            for _ in range(args.reps):
                t0 = time.perf_counter(); call_packed(); eng.synchronize(); packed.append((time.perf_counter() - t0) * 1e3)
    for step in STEPS:
        traffic = npts * (step + 16)
        ku, cu = float(np.median(unpack[step])), float(np.median(copy[step]))
        emit({"record": "unpack", "frames": F, "points": npts, "step": step, "traffic_bytes": traffic, "kernel_us_median": round(ku, 1),
              "kernel_GBps": round(traffic / ku / 1e3, 1), "memcpy_bytes": traffic // 2, "memcpy_us_median": round(cu, 1),
              "memcpy_GBps": round(traffic / cu / 1e3, 1), "kernel_over_memcpy": round(ku / cu, 3), "samples": len(unpack[step])}, out)
    pm = float(np.median(packed))
    for step in STEPS:
        sm = float(np.median(steps[step]))
        emit({"record": "device_batch", "frames": F, "points": npts, "step": step, "records_step_ms_median": round(sm, 3),
              "packed_float4_step_ms_median": round(pm, 3), "difference_ms": round(sm - pm, 3),
              "unpack_kernel_ms_median": round(float(np.median(unpack[step])) / 1e3, 3), "samples": len(steps[step])}, out)
    eng.close()


def host_legs(args, out):
    tmp = tempfile.mkdtemp(prefix="pwpp_records_bench_")
    exe = os.path.join(tmp, "pc2_latency")
    lib_dir = os.path.join(PKG, "lib")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tools", "pc2_latency.cpp"), "-o", exe,
                           "-L" + lib_dir, "-lpwpp_b200", "-Wl,-rpath," + lib_dir])
    z = np.load(os.path.join(REPO, "tests", "golden", "kitti_000000.npz"))
    scan = os.path.join(tmp, "scan.bin")
    np.ascontiguousarray(z["xyzi_t"].T, dtype=np.float32).tofile(scan)
    for name in ("pcl_xyzi32", "velodyne22", "rec48"):
        res = subprocess.run([exe, scan, name, str(args.host_reps)], capture_output=True, text=True, timeout=1200)
        assert res.returncode == 0, res.stderr
        for line in res.stdout.splitlines():
            if line.startswith("{"):
                rec = json.loads(line)
                rec["points"] = int(z["xyzi_t"].shape[1])
                emit(rec, out)


def bench_legs(args, out):
    trees = [("this", REPO)] + ([("parent", os.path.abspath(args.parent))] if args.parent else [])
    for rnd in range(3):
        for tag, tree in trees:
            res = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", "10", "--warmup", "3"], capture_output=True,
                                 text=True, cwd=tree, timeout=3600)
            assert res.returncode == 0, res.stderr[-2000:]
            line = [l for l in res.stdout.splitlines() if l.startswith("{")][-1]
            b = json.loads(line)
            emit({"record": "bench", "tree": tag, "run": rnd, "line": b}, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--parent", default="", help="the parent commit's tree, built, for the bench.py A/B")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-reps", type=int, default=300)
    ap.add_argument("--legs", default="unpack,host,bench")
    args = ap.parse_args()
    import stream_map_bench
    emit(stream_map_bench.gpu_info(), args.out)
    legs = args.legs.split(",")
    if "unpack" in legs:
        device_legs(args, args.out)
    if "host" in legs:
        host_legs(args, args.out)
    if "bench" in legs:
        bench_legs(args, args.out)
    emit(stream_map_bench.gpu_info(), args.out)


if __name__ == "__main__":
    main()
