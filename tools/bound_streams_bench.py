"""What a stream table costs and saves (pwpp_bind_stream_table). One JSON line per record on stdout and in --out. Run on the GPU
from the repository root after build():

  python tools/bound_streams_bench.py [--out FILE]

  gpu       card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  fleet     256 streams with default Params served by a 64-position bound call over 16-byte KITTI records (the six fixture scans
            cycled); a seeded scheduler picks 64 of the 256 streams per tick from 32 precomputed schedules, copied in device to
            device before each replay. (a) stream_table: one ctx of 256 streams, the pick copied into d_streams; (b) slot_swap: a
            ctx of 64 slot streams and a 256-row device blob store, the picked rows gathered, imported, run, exported and
            scattered back, all in one graph; (c) rebind: unbind, bind the picked streams and run, host clock (for scale only).
            (a) and (b) must give identical index lists on the first tick before anything is timed. Device time between CUDA
            events around the copy and one replay, median of --reps, three alternated runs.
  overhead  one-frame and 64-frame replays with a stream table equal to the bound streams, against the same bind without one
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
from state_copy_bench import scan  # noqa: E402

SEED = 20261018
F, NS, K = 64, 256, 32


def data64():
    import torch
    scans = [scan(k) for k in range(6)]
    data = [torch.as_tensor(scans[f % 6], device="cuda").contiguous() for f in range(F)]
    return data, [len(scans[f % 6]) for f in range(F)]


def graph_of(fn, st):
    import torch
    with torch.cuda.stream(st):
        for _ in range(3):
            fn(st.cuda_stream)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return g


def fleet_leg(args, out):
    import torch
    import pwpp_b200
    data, sizes = data64()
    lay = layout16()
    counts = torch.tensor(sizes, dtype=torch.int64, device="cuda")
    rng = np.random.default_rng(SEED)
    sched = torch.tensor(np.stack([rng.permutation(NS)[:F] for _ in range(K)]), dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    # (a) the stream table
    a = pwpp_b200.Engine(device=0, num_streams=NS)
    pick = sched[0].clone()
    a.bind_call([d.data_ptr() for d in data], sizes, [lay] * F, counts, streams=list(range(F)))
    a.bind_stream_table(pick)
    # (b) 64 slot streams and a blob store of the 256 streams
    b = pwpp_b200.Engine(device=0, num_streams=F)
    b.bind_call([d.data_ptr() for d in data], sizes, [lay] * F, counts)
    stride = (b.state_blob_size() + 15) // 16 * 16
    store, _ = b.export_states([0] * NS)   # 256 constructor-state blobs (all 64 slots are fresh)
    torch.cuda.synchronize()
    store = store.clone()
    rows = torch.empty((F, stride), dtype=torch.uint8, device="cuda")
    slots = torch.arange(F, dtype=torch.int32, device="cuda")
    pick_b = sched[0].clone()

    def swap_tick(cs):
        torch.index_select(store, 0, pick_b.long(), out=rows)
        b.import_states(rows, slots, stream=cs)
        b.run_bound_call(cs)
        b.export_states(slots, out=rows, stream=cs)
        store.index_copy_(0, pick_b.long(), rows)

    # the first tick, eager, both ways: identical index lists
    a.run_bound_call(st.cuda_stream)
    with torch.cuda.stream(st):
        swap_tick(st.cuda_stream)
    st.synchronize()
    ia, oa, _, _ = a.bound_call_results()
    ib, ob, _, _ = b.bound_call_results()
    torch.cuda.synchronize()
    assert torch.equal(oa, ob) and torch.equal(ia[:int(oa[-1])], ib[:int(ob[-1])]), "stream table and slot swap differ on the first tick"
    emit({"record": "fleet_check", "first_tick_index_lists_identical": True, "points": int(oa[-1])}, out)
    graphs = {"stream_table": (graph_of(a.run_bound_call, st), pick), "slot_swap": (graph_of(swap_tick, st), pick_b)}
    step = {"k": 0}

    def replay(name):
        g, dst = graphs[name]

        def fn():
            k = step["k"] = (step["k"] + 1) % K
            with torch.cuda.stream(st):
                dst.copy_(sched[k], non_blocking=True)
                g.replay()
        return fn

    for name in graphs:
        for _ in range(K):
            replay(name)()
    st.synchronize()
    for rnd in range(3):
        for name in (list(graphs) if rnd % 2 == 0 else list(graphs)[::-1]):
            h, d = timed(replay(name), args.reps, st)
            emit({"record": "fleet", "path": name, "run": rnd, "frames": F, "streams": NS, "schedules": K, "seed": SEED,
                  "host_us_median": round(h, 1), "device_us_median": round(d, 1), "reps": args.reps}, out)
    a.unbind_call()
    b.unbind_call()
    b.close()
    # (c) rebinding per tick, host clock
    times = []
    picks = sched.cpu().numpy()
    for k in range(args.rebind_reps):
        t0 = time.perf_counter()
        a.bind_call([d.data_ptr() for d in data], sizes, [lay] * F, counts, streams=picks[k % K])
        a.run_bound_call(st.cuda_stream)
        st.synchronize()
        a.unbind_call()
        times.append((time.perf_counter() - t0) * 1e6)
    emit({"record": "fleet", "path": "rebind", "frames": F, "streams": NS, "host_us_median": round(float(np.median(times)), 1),
          "reps": args.rebind_reps}, out)
    a.close()


def overhead_leg(args, out):
    import torch
    import pwpp_b200
    data, sizes = data64()
    lay = layout16()
    st = torch.cuda.Stream()
    for nf in (1, F):
        counts = torch.tensor(sizes[:nf], dtype=torch.int64, device="cuda")
        graphs, engines = {}, []
        for name in ("no_table", "identity_table"):
            e = pwpp_b200.Engine(device=0, num_streams=nf)
            e.bind_call([d.data_ptr() for d in data[:nf]], sizes[:nf], [lay] * nf, counts)
            if name == "identity_table":
                t = torch.arange(nf, dtype=torch.int32, device="cuda")
                e.bind_stream_table(t)
            graphs[name] = graph_of(e.run_bound_call, st)
            engines.append(e)

        def replay(g):
            def fn():
                with torch.cuda.stream(st):
                    g.replay()
            return fn

        for g in graphs.values():
            for _ in range(20):
                replay(g)()
        st.synchronize()
        for rnd in range(3):
            for name in (list(graphs) if rnd % 2 == 0 else list(graphs)[::-1]):
                h, d = timed(replay(graphs[name]), args.reps, st)
                emit({"record": "overhead", "path": name, "run": rnd, "frames": nf, "host_us_median": round(h, 1),
                      "device_us_median": round(d, 1), "reps": args.reps}, out)
        for e in engines:
            e.unbind_call()
            e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rebind-reps", type=int, default=10)
    ap.add_argument("--legs", default="fleet,overhead")
    args = ap.parse_args()
    import stream_map_bench
    emit(stream_map_bench.gpu_info(), args.out)
    legs = args.legs.split(",")
    if "fleet" in legs:
        fleet_leg(args, args.out)
    if "overhead" in legs:
        overhead_leg(args, args.out)


if __name__ == "__main__":
    main()
