"""What reading scans in place from rings saves (pwpp_bind_call_rings). One JSON line per record on stdout and in --out; the card's
name, power limit and clocks come first and last. Run on the GPU from the repository root after build():

  python tools/bound_rings_bench.py [--parent DIR] [--out FILE]

  ragged    64 KITTI-shaped sensors (the six fixture scans cycled) on 3-slot rings, in 16-byte (x, y, z, intensity) and 22-byte
            (velodyne: + ring, time) records, with bound_actions_bench.py's seeded schedule that drops 10 % of the frames. Every
            tick the producer writes the next scan of every present sensor into slot (t + 1) % 3 of its ring (one device gather
            kernel from a staging copy, the same in both paths). Then either (copy) one index_select kernel copies every
            sensor's newest slot into fixed buffers bound with pwpp_bind_call_actions and that call's graph is replayed, or (ring)
            the ring-bound call's graph is replayed with the slots published in a device tensor. Both write the tick's actions
            (and slots) from a precomputed device table first. Device time between CUDA events around the tick, median of
            --reps ticks, three alternated runs with the order flipped, the SM clock sampled in every window. Before timing, both
            paths run the same 32 ticks side by side on fresh contexts and their device results (indices, offsets, num_ground,
            status) must be equal at every tick
  one_frame the same for one KITTI frame (16-byte records, no drops)
  bench     bench.py --gpus 1 --steps 10 --warmup 3 of this tree and of the parent tree --parent, alternated (the benchmarked path
            does not run the ring code)
"""
import argparse
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, "patchwork-plusplus_b200")
for p in (os.path.join(REPO, "tools"), PKG, os.path.join(PKG, "lib"), REPO):
    if p not in sys.path:
        sys.path.insert(0, p)

from bound_actions_bench import SEED, bench_legs, rounds, scan, timed_with_clocks  # noqa: E402
from bound_call_bench import emit  # noqa: E402

R = 3    # slots per ring
K = 32   # schedules cycled through the timed ticks
VELODYNE22 = np.dtype({"names": ["x", "y", "z", "intensity", "ring", "time"], "formats": ["<f4"] * 4 + ["<u2", "<f4"],
                       "offsets": [0, 4, 8, 12, 16, 18], "itemsize": 22})


def as_records(a, step):
    if step == 16:
        return np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    r = np.zeros(len(a), VELODYNE22)
    for c, nm in enumerate(("x", "y", "z", "intensity")):
        r[nm] = a[:, c]
    r["ring"] = np.arange(len(a)) % 64
    r["time"] = np.arange(len(a), dtype=np.float32) * 1e-6
    return r.view(np.uint8).reshape(-1)


def rings_leg(args, out, F, step, drop, record):
    import torch
    import pwpp_b200
    lay = pwpp_b200.layout_from_dtype(np.dtype({"names": ["x", "y", "z", "intensity"], "formats": ["<f4"] * 4, "offsets": [0, 4, 8, 12],
                                                "itemsize": 16}) if step == 16 else VELODYNE22)
    scans = [scan(k) for k in range(6)]
    sizes = [len(scans[f % 6]) for f in range(F)]
    sb = (max(sizes) * step + 15) // 16 * 16          # bytes of a slot (and of a fixed buffer)
    staging = torch.zeros(F, sb, dtype=torch.uint8, device="cuda")
    for f in range(F):
        rec = as_records(scans[f % 6], step)
        staging[f, :len(rec)] = torch.from_numpy(rec.copy()).cuda()
    ring_all = torch.zeros(R, F, sb, dtype=torch.uint8, device="cuda")   # slot s of sensor f: ring_all[s, f]
    for s in range(R):
        ring_all[s].copy_(staging)
    flat = ring_all.view(R * F, sb)
    counts_all = torch.tensor([[n] * R for n in sizes], dtype=torch.int64, device="cuda")   # ring f's counts: counts_all[f]
    bufs = torch.zeros(F, sb, dtype=torch.uint8, device="cuda")
    counts = torch.tensor(sizes, dtype=torch.int64, device="cuda")
    # the schedule: actions per tick, every present sensor's newest slot moves on, the producer writes that slot
    rng = np.random.default_rng(SEED)
    acts = np.where(rng.random((K, F)) < drop, pwpp_b200.FRAME_SKIP, pwpp_b200.FRAME_RUN).astype(np.int32)
    cur = np.zeros((K, F), np.int32)
    c = np.zeros(F, np.int32)
    for k in range(K):
        c = np.where(acts[k] == pwpp_b200.FRAME_RUN, (c + 1) % R, c)
        cur[k] = c
    d_acts, d_cur = torch.from_numpy(acts).cuda(), torch.from_numpy(cur).cuda()
    rows = torch.from_numpy((cur.astype(np.int64) * F + np.arange(F)[None, :])).cuda()                  # newest slot rows of flat
    wrows = [torch.from_numpy((cur[k].astype(np.int64) * F + np.arange(F))[acts[k] == pwpp_b200.FRAME_RUN]).cuda() for k in range(K)]
    wsrc = [torch.from_numpy(np.flatnonzero(acts[k] == pwpp_b200.FRAME_RUN)).cuda() for k in range(K)]
    st = torch.cuda.Stream()

    def contexts():
        actions, slots = torch.zeros(F, dtype=torch.int32, device="cuda"), torch.zeros(F, dtype=torch.int32, device="cuda")
        copy_e, ring_e = pwpp_b200.Engine(device=0, num_streams=F), pwpp_b200.Engine(device=0, num_streams=F)
        copy_e.bind_call([bufs[f].data_ptr() for f in range(F)], sizes, [lay] * F, counts, actions=actions)
        rings = [(ring_all.view(-1)[f * sb:], counts_all[f], F * sb) for f in range(F)]
        ring_e.bind_call_rings(rings, sizes, [lay] * F, slots, actions=actions)
        bufs.copy_(ring_all[0])   # the warm-up runs below read the same scans in both paths (slot 0)
        torch.cuda.synchronize()
        graphs = {}
        with torch.cuda.stream(st):
            for name, e in (("copy", copy_e), ("ring", ring_e)):
                for _ in range(2):
                    e.run_bound_call(st.cuda_stream)
                st.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    e.run_bound_call(torch.cuda.current_stream().cuda_stream)
                graphs[name] = g
        torch.cuda.synchronize()
        return actions, slots, (copy_e, ring_e), graphs

    def produce(k):   # the producer's write of the next scan of every present sensor, the same in both paths
        if len(wsrc[k]):
            flat.index_copy_(0, wrows[k], staging.index_select(0, wsrc[k]))

    def ticks(actions, slots, graphs):
        step_ = {"copy": 0, "ring": 0}

        def copy_tick():
            k = step_["copy"] = (step_["copy"] + 1) % K
            with torch.cuda.stream(st):
                produce(k)
                actions.copy_(d_acts[k], non_blocking=True)
                torch.index_select(flat, 0, rows[k], out=bufs)
                graphs["copy"].replay()

        def ring_tick():
            k = step_["ring"] = (step_["ring"] + 1) % K
            with torch.cuda.stream(st):
                produce(k)
                actions.copy_(d_acts[k], non_blocking=True)
                slots.copy_(d_cur[k], non_blocking=True)
                graphs["ring"].replay()
        return {"copy_newest_slots_then_replay": copy_tick, "ring_replay": ring_tick}

    # outputs compared between the paths: the same ticks side by side on contexts that saw the same warm-up runs
    actions, slots, engs, graphs = contexts()
    legs = ticks(actions, slots, graphs)
    for k in range(K):
        for name, e in zip(legs, engs):
            legs[name]()
            st.synchronize()
            res = [t.clone() for t in e.bound_call_results()]
            if name.startswith("copy"):
                ref = res
            else:
                assert all(torch.equal(a, b) for a, b in zip(ref, res)), f"tick {k}: the ring replay differs from copy + replay"
    for rnd, names in rounds(list(legs)):
        for name in names:
            h, d, clk = timed_with_clocks(legs[name], args.reps, st)
            emit({"record": record, "path": name, "run": rnd, "frames": F, "point_step": step, "slots": R, "drop": drop, "seed": SEED,
                  "schedules": K, "host_us_median": round(h, 1), "device_us_median": round(d, 1), "reps": args.reps, "clocks": clk}, out)
    for e in engs:
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--parent", default="", help="the parent commit's tree, built, for the bench.py A/B")
    ap.add_argument("--reps", type=int, default=150)
    ap.add_argument("--bench-runs", type=int, default=2)
    ap.add_argument("--legs", default="ragged,one_frame,bench")
    args = ap.parse_args()
    import stream_map_bench
    emit(stream_map_bench.gpu_info(), args.out)
    legs = args.legs.split(",")
    if "ragged" in legs:
        for step in (16, 22):
            rings_leg(args, args.out, 64, step, 0.10, "ragged")
    if "one_frame" in legs:
        rings_leg(args, args.out, 1, 16, 0.0, "one_frame")
    if "bench" in legs:
        bench_legs(args, args.out)
    emit(stream_map_bench.gpu_info(), args.out)


if __name__ == "__main__":
    main()
