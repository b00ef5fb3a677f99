"""What stream state on the GPU costs (pwpp_export_states_device / pwpp_import_states_device / pwpp_clone). One JSON line per record on
stdout and in --out. Run on the GPU from the repository root after build():

  python tools/state_copy_bench.py [--out FILE]

  gpu        card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  migrate    64 streams with default Params (history capacity 1280: 82,112 bytes per stream blob, 5.3 MB for all 64), each after
             a few KITTI frames (history rows are copied whole, so the volume does not depend on how full they are): one device
             export of all 64 plus one device import of all 64 (CUDA events around both, median of --reps), against the host loop
             of pwpp_export_state + pwpp_import_state over the 64 streams (host clock, median of --host-reps)
  copy       what `PatchWorkpp b = a;` costs: pwpp_clone of a one-stream ctx after one KITTI frame, against constructing a fresh
             instance (pwpp_create + pwpp_set_output_order, what the drop-in constructor calls); host clock, medians of --copy-reps,
             alternated
  tick       a 64-sensor bound tick (the six fixture scans cycled as 16-byte records) as a CUDA graph: the bare run, against the
             run with a device export of every stream before it and an import after it whose stream list is computed on the GPU
             from a rollback mask (about 10 % of the streams rolled back per tick, seeded schedule copied in device to device);
             device time between CUDA events around one replay, median of --reps, three alternated runs
"""
import argparse
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, "patchwork-plusplus_b200")
for p in (os.path.join(REPO, "tools"), PKG, os.path.join(PKG, "lib"), REPO):
    if p not in sys.path:
        sys.path.insert(0, p)

from bound_call_bench import emit, layout16, timed  # noqa: E402

SEED = 20261018
F = 64


def scan(k):
    z = np.load(os.path.join(REPO, "tests", "golden", f"kitti_{k:06d}.npz"))
    return np.ascontiguousarray(z["xyzi_t"].T, dtype=np.float32)


def migrate_leg(args, out):
    import torch
    import pwpp_b200
    scans = [scan(k) for k in range(6)]
    e = pwpp_b200.Engine(device=0, num_streams=F)
    for r in range(3):
        e.estimate_host([scans[(f + r) % 6] for f in range(F)])
    e.synchronize()
    st = torch.cuda.Stream()
    ids = torch.arange(F, dtype=torch.int32, device="cuda")
    blob = int(e.lib.pwpp_stream_state_blob_size(e._h, 0))
    rows = torch.empty((F, (e.state_blob_size() + 15) // 16 * 16), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def device_pair():
        e.export_states(ids, out=rows, stream=st.cuda_stream)
        e.import_states(rows, ids, stream=st.cuda_stream)

    for _ in range(20):
        device_pair()
    st.synchronize()
    _, d = timed(device_pair, args.reps, st)

    def host_loop():
        for s in range(F):
            e.import_state(s, e.export_state(s))

    host_loop()
    host = []
    for _ in range(args.host_reps):
        t0 = time.perf_counter()
        host_loop()
        host.append((time.perf_counter() - t0) * 1e6)
    mb = 2 * F * blob / 1e6
    emit({"record": "migrate", "streams": F, "blob_bytes": blob, "bytes_each_way": F * blob, "device_export_plus_import_us_median": round(d, 1),
          "device_reps": args.reps, "device_GBps_read_plus_write": round(2 * mb / d * 1e6 / 1e3, 1),
          "host_loop_us_median": round(float(np.median(host)), 1), "host_reps": args.host_reps}, out)
    e.close()


def copy_leg(args, out):
    import pwpp_b200
    a = pwpp_b200.Engine(device=0)
    a.set_output_order(1)
    a.estimate_host([scan(0)])

    def clone():
        a.clone().close()

    def fresh():
        e = pwpp_b200.Engine(device=0)
        e.set_output_order(1)
        e.close()

    legs = {"clone_after_one_frame": clone, "fresh_instance": fresh}
    for fn in legs.values():
        for _ in range(3):
            fn()
    res = {k: [] for k in legs}
    for rnd in range(args.copy_reps):
        for name in (list(legs) if rnd % 2 == 0 else list(legs)[::-1]):
            t0 = time.perf_counter()
            legs[name]()
            res[name].append((time.perf_counter() - t0) * 1e6)
    for name, v in res.items():
        emit({"record": "copy", "path": name, "host_us_median": round(float(np.median(v)), 1), "reps": args.copy_reps}, out)
    a.close()


def tick_leg(args, out):
    import torch
    import pwpp_b200
    scans = [scan(k) for k in range(6)]
    data = [torch.from_numpy(scans[f % 6]).cuda().view(torch.uint8).reshape(-1).clone() for f in range(F)]
    sizes = [len(scans[f % 6]) for f in range(F)]
    lay = layout16()
    counts = torch.tensor(sizes, dtype=torch.int64, device="cuda")
    rng = np.random.default_rng(SEED)
    K = 32
    table = torch.from_numpy(rng.random((K, F)) < 0.10).cuda()
    mask = torch.zeros(F, dtype=torch.bool, device="cuda")
    ids = torch.arange(F, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    engines, graphs = {}, {}
    for name in ("bare_tick", "tick_with_snapshot_and_rollback"):
        e = pwpp_b200.Engine(device=0, num_streams=F)
        e.bind_call([d.data_ptr() for d in data], sizes, [lay] * F, counts)
        engines[name] = e
    rows = torch.empty((F, (engines["bare_tick"].state_blob_size() + 15) // 16 * 16), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        for name, e in engines.items():
            for _ in range(3):
                e.run_bound_call(st.cuda_stream)
            st.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                cs = torch.cuda.current_stream().cuda_stream
                if name == "bare_tick":
                    e.run_bound_call(cs)
                else:
                    e.export_states(ids, out=rows, stream=cs)
                    e.run_bound_call(cs)
                    restore = torch.where(mask, ids, torch.full_like(ids, -1))   # the rollback decision, on the GPU
                    e.import_states(rows, restore, stream=cs)
            graphs[name] = g
    torch.cuda.synchronize()
    step = {"k": 0}

    def replay(g):
        def fn():
            k = step["k"] = (step["k"] + 1) % K
            with torch.cuda.stream(st):
                mask.copy_(table[k], non_blocking=True)
                g.replay()
        return fn

    for g in graphs.values():
        for _ in range(K):
            replay(g)()
    st.synchronize()
    for rnd in range(3):
        for name in (list(graphs) if rnd % 2 == 0 else list(graphs)[::-1]):
            h, d = timed(replay(graphs[name]), args.reps, st)
            emit({"record": "tick", "path": name, "run": rnd, "frames": F, "rollback_fraction": 0.10, "seed": SEED,
                  "host_us_median": round(h, 1), "device_us_median": round(d, 1), "reps": args.reps}, out)
    for e in engines.values():
        e.unbind_call()
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--host-reps", type=int, default=10)
    ap.add_argument("--copy-reps", type=int, default=20)
    ap.add_argument("--legs", default="migrate,copy,tick")
    args = ap.parse_args()
    import stream_map_bench
    emit(stream_map_bench.gpu_info(), args.out)
    legs = args.legs.split(",")
    if "migrate" in legs:
        migrate_leg(args, args.out)
    if "copy" in legs:
        copy_leg(args, args.out)
    if "tick" in legs:
        tick_leg(args, args.out)
    emit(stream_map_bench.gpu_info(), args.out)


if __name__ == "__main__":
    main()
