"""What a width ladder (pwpp_bind_width_ladder) saves when the GPU, not the host, knows how many sensors arrived. One JSON line
per record on stdout and in --out. Run on the GPU from the repository root after build():

  python tools/bound_ladder_bench.py [--out FILE]

  gpu       card name, power limit and maximum SM clock (nvidia-smi), read in the same command as the numbers
  check     for every k, one tick through (a), (b) and (c) on three contexts of identical history: identical index lists and
            offsets over the k present positions ((b) and (c): over all 64, with the same status), before anything is timed
  tick      bound_calls_bench.py's fleet: 256 streams with default Params over 16-byte KITTI records (the six fixture scans
            cycled); a tick holds k present sensors, k in {1, 4, 16, 64}, picked by a seeded scheduler from 32 precomputed
            schedules and copied device to device into a stream table before each replay. (a) buckets: one ctx with four bound
            calls of 1, 4, 16 and 64 positions, the host replaying the smallest that holds k; (b) holes: the 64-position
            stream-table graph, positions k .. 63 set to -1; (c) ladder: the same 64-position call with the width ladder
            {1, 4, 16}, the same holes, one graph whose width the GPU picks. Device time between CUDA events around the copy and
            one replay, median of --reps, three alternated runs.
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

from bound_call_bench import emit, layout16, timed  # noqa: E402
from bound_calls_bench import BUCKETS, F, K, NS, SEED  # noqa: E402
from bound_streams_bench import data64, graph_of  # noqa: E402

LADDER = [1, 4, 16]
WAYS = ("buckets", "holes", "ladder")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    import torch
    import pwpp_b200
    import stream_map_bench
    out = args.out
    emit(stream_map_bench.gpu_info(), out)
    data, sizes = data64()
    lay = layout16()
    counts = torch.tensor(sizes, dtype=torch.int64, device="cuda")
    rng = np.random.default_rng(SEED)
    sched = torch.tensor(np.stack([rng.permutation(NS)[:F] for _ in range(K)]), dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    # (a) one ctx, bound calls 0..3 of 1, 4, 16 and 64 positions, bound widest first so that every buffer grows once
    a = pwpp_b200.Engine(device=0, num_streams=NS)
    picks = {}
    for i in reversed(range(len(BUCKETS))):
        k = BUCKETS[i]
        a.select_bound_call(i)
        a.bind_call([d.data_ptr() for d in data[:k]], sizes[:k], [lay] * k, counts[:k], streams=list(range(k)))
        picks[k] = sched[0, :k].clone()
        a.bind_stream_table(picks[k])
    # (b) the 64-position stream-table call alone, holes past k; (c) the same call with the ladder
    b, c = pwpp_b200.Engine(device=0, num_streams=NS), pwpp_b200.Engine(device=0, num_streams=NS)
    pick = {}
    for name, e in (("holes", b), ("ladder", c)):
        e.bind_call([d.data_ptr() for d in data], sizes, [lay] * F, counts, streams=list(range(F)))
        pick[name] = sched[0].clone()
        e.bind_stream_table(pick[name])
    c.bind_width_ladder(LADDER)
    holes = {k: torch.cat([sched[:, :k], torch.full((K, F - k), -1, dtype=torch.int32, device="cuda")], 1) for k in BUCKETS}

    def run_a(i):
        def fn(cs):
            a.select_bound_call(i)
            a.run_bound_call(cs)
        return fn

    # one tick of every k through all three, eager, in the same order on every context: identical lists
    for i, k in enumerate(BUCKETS):
        picks[k].copy_(sched[i, :k])
        pick["holes"].copy_(holes[k][i])
        pick["ladder"].copy_(holes[k][i])
        torch.cuda.synchronize()
        run_a(i)(st.cuda_stream)
        b.run_bound_call(st.cuda_stream)
        c.run_bound_call(st.cuda_stream)
        st.synchronize()
        a.select_bound_call(i)
        ia, oa, _, sa = a.bound_call_results()
        ib, ob, _, sb = b.bound_call_results()
        ic, oc, _, sc = c.bound_call_results()
        torch.cuda.synchronize()
        assert torch.equal(oa, ob[:k + 1]) and int(ob[-1]) == int(ob[k]), f"k={k}: offsets differ"
        assert torch.equal(ia[:int(oa[-1])], ib[:int(ob[-1])]), f"k={k}: index lists differ"
        assert torch.equal(ob, oc) and torch.equal(sb, sc) and torch.equal(ib[:int(ob[-1])], ic[:int(oc[-1])]), f"k={k}: the ladder differs"
        assert int(sa.abs().sum()) == 0 and int(sb[:k].abs().sum()) == 0, f"k={k}: a present position was rejected"
        width = int(c.bound_call_width().item())
        assert width == min(w for w in LADDER + [F] if w >= k), f"k={k}: width {width}"
        emit({"record": "check", "k": k, "index_lists_identical": True, "points": int(oa[-1]), "ladder_width": width}, out)

    graphs_a = {k: graph_of(run_a(i), st) for i, k in enumerate(BUCKETS)}
    graph = {"holes": graph_of(b.run_bound_call, st), "ladder": graph_of(c.run_bound_call, st)}
    step = {"t": 0}

    def tick(way, k):
        def fn():
            t = step["t"] = (step["t"] + 1) % K
            with torch.cuda.stream(st):
                if way == "buckets":
                    picks[k].copy_(sched[t, :k], non_blocking=True)
                    graphs_a[k].replay()
                else:
                    pick[way].copy_(holes[k][t], non_blocking=True)
                    graph[way].replay()
        return fn

    for k in BUCKETS:
        for way in WAYS:
            for _ in range(K):
                tick(way, k)()
    st.synchronize()
    for rnd in range(3):
        for k in BUCKETS:
            for way in (WAYS if rnd % 2 == 0 else WAYS[::-1]):
                h, d = timed(tick(way, k), args.reps, st)
                emit({"record": "tick", "way": way, "k": k, "graph_positions": k if way == "buckets" else F, "run": rnd,
                      "streams": NS, "schedules": K, "seed": SEED, "host_us_median": round(h, 1), "device_us_median": round(d, 1),
                      "reps": args.reps}, out)
    emit(stream_map_bench.gpu_info(), out)
    for i in range(len(BUCKETS)):
        a.select_bound_call(i)
        a.unbind_call()
    for e in (b, c):
        e.unbind_call()
        e.close()
    a.close()


if __name__ == "__main__":
    main()
