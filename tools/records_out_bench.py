"""What returning the segmented clouds as the sensor's own records costs (pwpp_device_record_results / pwpp_host_record_results,
k_gather_records). One JSON line per record on stdout and in --out. Run on the GPU from the repository root after build():

  python tools/records_out_bench.py [--parent DIR] [--out FILE]

  gpu      card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  gather   the gather kernel alone (k_gather_records, kernel time from torch.profiler over --reps calls) on bench.py's
           1024-frame KITTI-64 batch laid out as records of 16, 22, 32 and 48 bytes (pwpp_estimate_device_records), in both
           output orders, next to a device-to-device copy with the same HBM traffic ((2 * step + 4) bytes per point: read the
           record and its index, write the record; a copy of step + 2 bytes per point), timed with CUDA events in the same run
  lists    what the source order costs: the same kernel as compiled for sm_90a (tests/gpu_records_gather_probe.cu, kernel time
           from torch.profiler over --list-reps launches) on the same batch and steps with four kinds of index list: identity
           (sequential sources, nothing dropped), the engine's own lists in bin order and in reference order, and each frame's
           points in a random order
  ros      one-frame latency of estimateGround(pw, message) plus both makeRecordsPayload calls against the same with both
           makeCloudPayload calls, kitti_000000 as pcl_xyzi32 and velodyne22, pageable and page-locked
           (tools/pc2_records_out_latency.cpp, built into a temporary directory)
  bench    bench.py --gpus 1 --steps 10 --warmup 3 of this tree and of the parent tree --parent (built), alternated, three runs each
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, "patchwork-plusplus_b200")
for p in (os.path.join(REPO, "tools"), PKG, os.path.join(PKG, "lib"), REPO):
    if p not in sys.path:
        sys.path.insert(0, p)

import records_bench  # noqa: E402  (make_records, layout, emit, bench_legs)

STEPS = records_bench.STEPS
emit = records_bench.emit


def gather_legs(args, out):
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
    recs = {}
    for step in STEPS:
        r = records_bench.make_records(pts, step)
        recs[step] = (r, (C.c_void_p * F)(*[r.data_ptr() + int(o) * step for o in offs_np[:-1]]),
                      (pwpp_b200.PwppPointLayout * F)(*([records_bench.layout(step)] * F)))
    torch.cuda.synchronize()
    d_rec, h_off = C.c_void_p(), C.c_void_p()

    def call_and_gather(step):
        _, ptrs, lays = recs[step]
        assert lib.pwpp_estimate_device_records(eng._h, F, ids, ptrs, ns, lays, None) == 0, lib.pwpp_last_error()
        assert lib.pwpp_device_record_results(eng._h, C.byref(d_rec), C.byref(h_off)) == 0, lib.pwpp_last_error()

    kernel = {(s, o): [] for s in STEPS for o in (0, 1)}
    copy = {s: [] for s in STEPS}
    kept = {}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for order in (0, 1):   # warm every shape
        eng.set_output_order(order)
        for step in STEPS:
            for _ in range(2):
                call_and_gather(step)
            eng.synchronize()
    for rnd in range(3):   # variants alternate within the run
        for order in (0, 1):
            eng.set_output_order(order)
            for step in STEPS:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.reps):
                        call_and_gather(step)
                    eng.synchronize()
                ks = [e for e in prof.events() if "k_gather_records" in e.name and e.device_type.name == "CUDA"]
                assert len(ks) == args.reps, len(ks)
                kernel[(step, order)] += [e.device_time for e in ks]   # microseconds
                kept[step] = np.ctypeslib.as_array((C.c_int64 * (F + 1)).from_address(h_off.value)).copy()
        for step in STEPS:
            nbytes = npts * (step + 2)
            src = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            dst = torch.empty_like(src)
            dst.copy_(src)
            for _ in range(args.reps):
                ev0.record(); dst.copy_(src); ev1.record(); ev1.synchronize()
                copy[step].append(ev0.elapsed_time(ev1) * 1e3)
            del src, dst
    # spot check of the last call's output (step 48, reference order) against the index lists
    eng.synchronize()
    rec_t = torch.as_tensor(view_of(d_rec.value, int(kept[STEPS[-1]][-1]), "|u1"), device="cuda")
    d_idx = C.c_void_p()
    assert lib.pwpp_device_results(eng._h, C.byref(d_idx), None) == 0
    idx = torch.as_tensor(view_of(d_idx.value, npts, "<i4"), device="cuda")
    r = recs[STEPS[-1]][0]
    for f in (0, F // 2, F - 1):
        o, n = int(offs_np[f]), int(offs_np[f + 1] - offs_np[f])
        m = int(lib.pwpp_num_ground(eng._h, f) + lib.pwpp_num_nonground(eng._h, f))
        want = r[o:o + n][idx[o:o + m].long()].reshape(-1)
        got = rec_t[int(kept[STEPS[-1]][f]):int(kept[STEPS[-1]][f]) + m * STEPS[-1]]
        assert torch.equal(got, want), f"frame {f}"
    lists_leg(args, out, eng, recs, offs_np, call_and_gather, profile, ProfilerActivity)
    for order in (0, 1):
        for step in STEPS:
            traffic = npts * (2 * step + 4)
            ku, cu = float(np.median(kernel[(step, order)])), float(np.median(copy[step]))
            emit({"record": "gather", "order": ("bin", "reference")[order], "frames": F, "points": npts, "step": step, "traffic_bytes": traffic,
                  "kernel_us_median": round(ku, 1), "kernel_GBps": round(traffic / ku / 1e3, 1), "memcpy_bytes": traffic // 2,
                  "memcpy_us_median": round(cu, 1), "memcpy_GBps": round(traffic / cu / 1e3, 1), "kernel_over_memcpy": round(ku / cu, 3),
                  "samples": len(kernel[(step, order)])}, out)
    eng.close()


def lists_leg(args, out, eng, recs, offs_np, call_and_gather, profile, ProfilerActivity):
    import torch
    if "lists" not in args.legs.split(","):
        return
    F, lib = len(offs_np) - 1, eng.lib
    npts = int(offs_np[-1])
    ns = np.diff(offs_np).astype(np.int64)
    probe = C.CDLL(os.path.join(PKG, "lib", "libpwpp_records_gather_probe.so"))
    probe.probe_gather_records.argtypes = [C.c_int] + [C.c_void_p] * 7
    probe.probe_gather_records.restype = C.c_int
    kinds = {"identity": (np.concatenate([np.arange(k, dtype=np.int32) for k in ns]), np.zeros(F, np.int32))}
    for order, name in ((0, "bin"), (1, "reference")):
        eng.set_output_order(order)
        call_and_gather(STEPS[0])
        a, b, c = C.c_void_p(), C.c_void_p(), C.c_void_p()
        assert lib.pwpp_host_results(eng._h, C.byref(a), C.byref(b), C.byref(c)) == 0
        idx = np.ctypeslib.as_array((C.c_int32 * npts).from_address(a.value)).copy()
        nd = np.array([ns[f] - lib.pwpp_num_ground(eng._h, f) - lib.pwpp_num_nonground(eng._h, f) for f in range(F)], np.int32)
        kinds[name] = (idx, nd)
    rng = np.random.default_rng(0)
    kinds["shuffled"] = (np.concatenate([rng.permutation(k).astype(np.int32) for k in ns]), np.zeros(F, np.int32))
    times = {(s, k): [] for s in STEPS for k in kinds}
    for rnd in range(2):
        for step in STEPS:
            r, ptrs, _ = recs[step]
            steps = np.full(F, step, np.int32)
            roff = np.zeros(F + 1, np.int64)
            dst = torch.empty(int(((ns * step + 15) // 16 * 16).sum()), dtype=torch.uint8, device="cuda")
            for kind, (idx, nd) in kinds.items():
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.list_reps):
                        assert probe.probe_gather_records(F, ptrs, ns.ctypes.data, steps.ctypes.data, idx.ctypes.data, nd.ctypes.data,
                                                          dst.data_ptr(), roff.ctypes.data) == 0
                ks = [e for e in prof.events() if "k_gather_records" in e.name and e.device_type.name == "CUDA"]
                assert len(ks) == args.list_reps, len(ks)
                times[(step, kind)] += [e.device_time for e in ks]
                if kind == "identity" and rnd == 0:   # identity lists: the output is the input
                    o = int(roff[F // 2])
                    first = int(offs_np[F // 2])
                    assert torch.equal(dst[o:o + int(ns[F // 2]) * step], r[first:first + int(ns[F // 2])].reshape(-1))
            del dst
    for step in STEPS:
        for kind, (idx, nd) in kinds.items():
            m = npts - int(nd.sum())
            traffic = m * (2 * step + 4)
            ku = float(np.median(times[(step, kind)]))
            emit({"record": "gather_lists", "lists": kind, "frames": F, "points": npts, "listed": m, "step": step, "traffic_bytes": traffic,
                  "kernel_us_median": round(ku, 1), "kernel_GBps": round(traffic / ku / 1e3, 1), "samples": len(times[(step, kind)])}, out)


def view_of(ptr, n, typestr):
    class _View:   # __cuda_array_interface__ v3: torch.as_tensor wraps the memory without copying
        def __init__(self):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}
    return _View()


def ros_legs(args, out):
    tmp = tempfile.mkdtemp(prefix="pwpp_records_out_bench_")
    exe = os.path.join(tmp, "pc2_records_out_latency")
    lib_dir = os.path.join(PKG, "lib")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tools", "pc2_records_out_latency.cpp"),
                           "-o", exe, "-L" + lib_dir, "-lpwpp_b200", "-Wl,-rpath," + lib_dir])
    z = np.load(os.path.join(REPO, "tests", "golden", "kitti_000000.npz"))
    scan = os.path.join(tmp, "scan.bin")
    np.ascontiguousarray(z["xyzi_t"].T, dtype=np.float32).tofile(scan)
    for name in ("pcl_xyzi32", "velodyne22"):
        res = subprocess.run([exe, scan, name, str(args.host_reps)], capture_output=True, text=True, timeout=1200)
        assert res.returncode == 0, res.stderr
        for line in res.stdout.splitlines():
            if line.startswith("{"):
                rec = json.loads(line)
                rec["points"] = int(z["xyzi_t"].shape[1])
                emit(rec, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--parent", default="", help="the parent commit's tree, built, for the bench.py A/B")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-reps", type=int, default=300)
    ap.add_argument("--list-reps", type=int, default=5)
    ap.add_argument("--legs", default="gather,lists,ros,bench")
    args = ap.parse_args()
    import stream_map_bench
    emit(stream_map_bench.gpu_info(), args.out)
    legs = args.legs.split(",")
    if "gather" in legs:
        gather_legs(args, args.out)
    if "ros" in legs:
        ros_legs(args, args.out)
    if "bench" in legs:
        records_bench.bench_legs(args, args.out)
    emit(stream_map_bench.gpu_info(), args.out)


if __name__ == "__main__":
    main()
