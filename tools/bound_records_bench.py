"""What the record results of a bound call cost (pwpp_bind_record_results, k_gather_record_parts). One JSON line per record on stdout
and in --out. Run on the GPU from the repository root after build():

  python tools/bound_records_bench.py [--parent-lib SO] [--out FILE]

  gpu       card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  latency   one KITTI frame (kitti_000000) as 22-byte (velodyne) and 32-byte (PCL xyzi) records on the device: a CUDA-graph replay
            of the bound call with record results (both parts) against one without, alternated. Device time between CUDA events
            around one replay, median of --reps replays, three runs
  parts     bench.py's 1024-frame KITTI-64 batch as records of 16, 22, 32 and 48 bytes, run as a bound call with both parts
            enabled: k_gather_record_parts alone (kernel time from torch.profiler over --kreps runs), with capacities equal to
            the frame sizes and with every capacity 1.5 x the largest frame, alternated, three runs
  direct    the same batch through pwpp_estimate_device_records and pwpp_device_record_results: k_gather_records on the same
            lists (kernel time from torch.profiler), next to a device-to-device copy with the gather's HBM traffic ((2 * step + 4)
            bytes per listed point; a copy of step + 2 bytes per point), three runs; with --parent-lib, the parent commit's
            library (a libpwpp_b200.so) runs the same calls, alternated with this tree's
"""
import argparse
import ctypes as C
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, "patchwork-plusplus_b200")
for p in (os.path.join(REPO, "tools"), PKG, os.path.join(PKG, "lib"), REPO):
    if p not in sys.path:
        sys.path.insert(0, p)

import records_bench  # noqa: E402  (make_records, layout, emit)

STEPS = records_bench.STEPS
emit = records_bench.emit


def kernel_times(fn, reps, name, sync):
    """Device times (us) of every launch of kernel `name` over reps calls of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        sync()
    ks = [e.device_time for e in prof.events() if e.name.split("(")[0].endswith(name) and e.device_type.name == "CUDA"]
    assert len(ks) == reps, (name, len(ks), reps)
    return ks


def latency_leg(args, out):
    import torch
    import pwpp_b200
    z = np.load(os.path.join(REPO, "tests", "golden", "kitti_000000.npz"))
    pts = torch.from_numpy(np.ascontiguousarray(z["xyzi_t"].T, dtype=np.float32)).cuda()
    n = pts.shape[0]
    st = torch.cuda.Stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for step, name in ((22, "velodyne22"), (32, "pcl_xyzi32")):
        rec = records_bench.make_records(pts, step)
        lay = records_bench.layout(step)
        counts = torch.tensor([n], dtype=torch.int64, device="cuda")
        graphs, engines = {}, []
        for variant in ("without", "with_record_results"):
            e = pwpp_b200.Engine(device=0)
            e.bind_call([rec.data_ptr()], [n], [lay], counts)
            if variant != "without":
                e.bind_record_results()
            with torch.cuda.stream(st):
                for _ in range(3):
                    e.run_bound_call(st.cuda_stream)
                st.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    e.run_bound_call(torch.cuda.current_stream().cuda_stream)
            graphs[variant] = g
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
                emit({"record": "latency", "layout": name, "step": step, "variant": variant, "run": rnd, "points": n,
                      "device_us_median": round(float(np.median(dev)), 1), "reps": args.reps}, out)
        for e in engines:
            e.close()
        del graphs
        torch.cuda.synchronize()


def batch(dev):
    import bench
    import synth
    F = 1024
    pts, offs = synth.make_batch(bench.SEED, 0, F, "kitti64", dev)
    return pts, offs.numpy().astype(np.int64)


def parts_leg(args, out, pts, offs_np):
    import torch
    import pwpp_b200
    F = len(offs_np) - 1
    sizes = np.diff(offs_np)
    npts = int(offs_np[-1])
    cap_pad = int(sizes.max() * 3 // 2)
    counts = torch.from_numpy(sizes.copy()).cuda()
    for step in STEPS:
        # frame f at offs[f] * step of one buffer that ends one padded capacity after the last frame's start: every capacity is
        # readable memory, and only the counts are ever read
        big = torch.zeros((npts + cap_pad) * step, dtype=torch.uint8, device="cuda")
        big[: npts * step] = records_bench.make_records(pts, step).reshape(-1)
        ptrs = [big.data_ptr() + int(o) * step for o in offs_np[:-1]]
        lay = records_bench.layout(step)
        engines = {}
        for variant, max_n in (("capacity_equals_size", sizes.tolist()), ("capacity_1.5x_largest", [cap_pad] * F)):
            e = pwpp_b200.Engine(device=0, num_streams=F)
            e.bind_call(ptrs, max_n, [lay] * F, counts)
            e.bind_record_results()
            for _ in range(2):
                e.run_bound_call()
            e.synchronize()
            engines[variant] = (e, sum(int(k) for k in max_n))
        times = {v: [] for v in engines}
        for rnd in range(3):
            for variant, (e, _) in engines.items():
                times[variant] += kernel_times(e.run_bound_call, args.kreps, "k_gather_record_parts", e.synchronize)
        # the output of the last run against the lists: a few frames of the padded variant
        e = engines["capacity_1.5x_largest"][0]
        _, ng, off, cnt = e.bound_record_results()
        idx, poff, nground, _ = e.bound_call_results()
        src = big[: npts * step].reshape(npts, step)
        for f in (0, F // 2, F - 1):
            o, g, k = int(poff[f]), int(nground[f]), int(cnt[f, 1])
            want = src[o: o + int(sizes[f])][idx[o + g: o + g + k].long()].reshape(-1)
            assert torch.equal(ng[int(off[f]): int(off[f]) + k * step], want), f"step {step} frame {f}"
        listed = int(cnt.sum())
        traffic = listed * (2 * step + 4)
        for variant, (e, cap) in engines.items():
            ku = float(np.median(times[variant]))
            emit({"record": "parts", "variant": variant, "frames": F, "points": npts, "listed": listed, "capacity_points": cap, "step": step,
                  "traffic_bytes": traffic, "kernel_us_median": round(ku, 1), "kernel_GBps": round(traffic / ku / 1e3, 1),
                  "samples": len(times[variant])}, out)
            e.close()
        del big, engines
        torch.cuda.empty_cache()


def parent_engine(path, kw):
    """An Engine on the parent commit's library, which lacks the newer entry points: only those this leg calls are declared
    (with this tree's signatures)."""
    import pwpp_b200
    lib, ref = C.CDLL(path), pwpp_b200.load_library()
    for name in ("pwpp_create", "pwpp_destroy", "pwpp_num_bins", "pwpp_last_error", "pwpp_estimate_device_records", "pwpp_device_record_results",
                 "pwpp_num_ground", "pwpp_num_nonground", "pwpp_synchronize"):
        fn, r = getattr(lib, name), getattr(ref, name)
        fn.argtypes, fn.restype = r.argtypes, r.restype
    load = pwpp_b200.load_library
    pwpp_b200.load_library = lambda: lib   # an Engine keeps the library it was created with
    try:
        return pwpp_b200.Engine(**kw)
    finally:
        pwpp_b200.load_library = load


def direct_leg(args, out, pts, offs_np):
    import torch
    import pwpp_b200
    F = len(offs_np) - 1
    npts = int(offs_np[-1])
    kw = dict(device=0, num_streams=F, max_points_per_frame=int(np.diff(offs_np).max()))
    engines = {"this": pwpp_b200.Engine(**kw)}
    if args.parent_lib:
        engines["parent"] = parent_engine(os.path.abspath(args.parent_lib), kw)
    ids = (C.c_int32 * F)(*range(F))
    ns = (C.c_int64 * F)(*np.diff(offs_np).tolist())
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for step in STEPS:
        rec = records_bench.make_records(pts, step)
        ptrs = (C.c_void_p * F)(*[rec.data_ptr() + int(o) * step for o in offs_np[:-1]])
        lays = (pwpp_b200.PwppPointLayout * F)(*([records_bench.layout(step)] * F))
        torch.cuda.synchronize()

        def call_and_gather(e):
            d_rec, h_off = C.c_void_p(), C.c_void_p()
            assert e.lib.pwpp_estimate_device_records(e._h, F, ids, ptrs, ns, lays, None) == 0, e.lib.pwpp_last_error()
            assert e.lib.pwpp_device_record_results(e._h, C.byref(d_rec), C.byref(h_off)) == 0, e.lib.pwpp_last_error()
        for e in engines.values():
            for _ in range(2):
                call_and_gather(e)
            e.synchronize()
        times = {t: [] for t in engines}
        copy = []
        nbytes = npts * (step + 2)
        src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        dst = torch.empty_like(src)
        dst.copy_(src)
        for rnd in range(3):
            for tag, e in engines.items():
                times[tag] += kernel_times(lambda: call_and_gather(e), args.kreps, "k_gather_records", e.synchronize)
            for _ in range(args.kreps):
                ev0.record(); dst.copy_(src); ev1.record(); ev1.synchronize()
                copy.append(ev0.elapsed_time(ev1) * 1e3)
        del src, dst
        e = engines["this"]
        listed = sum(int(e.lib.pwpp_num_ground(e._h, f) + e.lib.pwpp_num_nonground(e._h, f)) for f in range(F))
        traffic = listed * (2 * step + 4)
        cu = float(np.median(copy))
        for tag in engines:
            ku = float(np.median(times[tag]))
            emit({"record": "direct", "library": tag, "frames": F, "points": npts, "listed": listed, "step": step, "traffic_bytes": traffic,
                  "kernel_us_median": round(ku, 1), "kernel_us_min": round(float(np.min(times[tag])), 1), "kernel_us_max": round(float(np.max(times[tag])), 1),
                  "kernel_GBps": round(traffic / ku / 1e3, 1), "memcpy_bytes": nbytes, "memcpy_us_median": round(cu, 1),
                  "samples": len(times[tag])}, out)
        del rec
        torch.cuda.empty_cache()
    for e in engines.values():
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--parent-lib", default="", help="the parent commit's libpwpp_b200.so, for the A/B of k_gather_records")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--kreps", type=int, default=10)
    ap.add_argument("--legs", default="latency,parts,direct")
    args = ap.parse_args()
    import torch
    import stream_map_bench
    emit(stream_map_bench.gpu_info(), args.out)
    legs = args.legs.split(",")
    if "latency" in legs:
        latency_leg(args, args.out)
    if "parts" in legs or "direct" in legs:
        pts, offs_np = batch(torch.device("cuda", 0))
        if "parts" in legs:
            parts_leg(args, args.out, pts, offs_np)
        if "direct" in legs:
            direct_leg(args, args.out, pts, offs_np)
    emit(stream_map_bench.gpu_info(), args.out)


if __name__ == "__main__":
    main()
