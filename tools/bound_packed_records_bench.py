"""What packed records of a bound call cost (pwpp_bind_packed_records, k_gather_record_packed) against the compaction a pipeline
needs around the capacity-layout record results today. One JSON line per record on stdout and, with --out FILE, in FILE. Run on
the GPU from the repository root after build():

  python tools/bound_packed_records_bench.py [--out FILE] [--reps R] [--runs K] [--kreps N]

  gpu     card name, power limit, maximum and current SM clock (nvidia-smi), read before and after the numbers in the same command
  tick    one tick of 64 KITTI-64 sensors in one packed batch (pwpp_bind_call_packed) as 22-byte velodyne and 16-byte float32
          xyzi records, whose consumer takes one packed non-ground record batch with device offsets, each form captured in one
          CUDA graph:
            today   capacity-layout non-ground record results (pwpp_bind_record_results), then a sync-free torch compaction: the
                    offsets from the device counts (cumsum), a gather of every capacity row (an index over the rows of an
                    overlapping (bytes, step) view) and an index_copy_ of the rows inside the counts into one packed (rows, step)
                    tensor;
            packed  packed non-ground records (pwpp_bind_packed_records).
          Device time between CUDA events around one replay, median of --reps replays, the two forms alternated, --runs runs.
          Before timing, both forms' packed records and offsets are checked equal byte for byte.
  kernel  bench.py's 1024-frame KITTI-64 batch bound with capacities equal to the sizes, as records of 16, 22, 32 and 48 bytes,
          record results and packed records both enabled (both parts): k_gather_record_packed against k_gather_record_parts
          from the same runs (kernel times from torch.profiler over --kreps runs), --runs runs. The packed output is checked
          against the capacity-layout output first.
"""
import argparse
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, "patchwork-plusplus_b200")
for p in (os.path.join(REPO, "tools"), PKG, os.path.join(PKG, "lib"), REPO):
    if p not in sys.path:
        sys.path.insert(0, p)

import records_bench  # noqa: E402  (make_records, layout, emit)

NF = 64
STEPS = records_bench.STEPS


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,driver_version"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, clk, cur, drv = [x.strip() for x in out[0].split(",")]
    return {"record": "gpu", "name": name, "power_limit": plim, "max_sm_clock": clk, "sm_clock": cur, "driver": drv}


def kitti_scans():
    d = os.path.join(REPO, "tests", "golden")
    names = sorted(f for f in os.listdir(d) if f.startswith("kitti_") and f.endswith(".npz"))
    return [np.ascontiguousarray(np.load(os.path.join(d, f))["xyzi_t"].T.astype(np.float32)) for f in names]


def kernel_times(fn, reps, names, sync):
    """Device times (us) of every launch of each kernel in `names` over reps calls of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        sync()
    out = {}
    for name in names:
        ks = [e.device_time for e in prof.events() if e.name.split("(")[0].endswith(name) and e.device_type.name == "CUDA"]
        assert len(ks) == reps, (name, len(ks), reps)
        out[name] = ks
    return out


class Today:
    """Capacity-layout record results, then a compaction with fixed shapes: every capacity row gathered (where each row starts
    is fixed by the layout), the rows inside the counts copied to their packed place, the rest to a spill row."""

    def __init__(self, pwpp_b200, points, offsets, max_n, lay, step):
        import torch
        self.eng = pwpp_b200.Engine(device=0, num_streams=NF)
        self.eng.bind_call_packed(points, offsets, list(max_n), layout=lay)
        self.eng.bind_record_results(False, True)
        _, self.ng, reg_off, self.cnt = self.eng.bound_record_results()
        cap = np.concatenate([[0], np.cumsum(max_n)])
        self.rows = int(cap[-1])
        fr = np.repeat(np.arange(NF), max_n)
        k = np.arange(self.rows) - cap[fr]
        self.src = torch.from_numpy((reg_off[fr] + k * step).astype(np.int64)).cuda()   # the first byte of every capacity row
        self.fr = torch.from_numpy(fr.astype(np.int64)).cuda()
        self.k = torch.from_numpy(k.astype(np.int64)).cuda()
        self.out = torch.zeros(self.rows + 1, step, dtype=torch.uint8, device="cuda")
        self.out_off = torch.zeros(NF + 1, dtype=torch.int64, device="cuda")

    def tick(self, stream):
        import torch
        step = self.out.shape[1]
        self.eng.run_bound_call(stream)
        c = self.cnt[:, 1].to(torch.int64)
        self.out_off[1:] = torch.cumsum(c, 0)
        dst = torch.where(self.k < c[self.fr], self.out_off[self.fr] + self.k, self.rows)
        self.out.index_copy_(0, dst, self.ng.unfold(0, step, 1)[self.src])


class Packed:
    def __init__(self, pwpp_b200, points, offsets, max_n, lay, step):
        self.eng = pwpp_b200.Engine(device=0, num_streams=NF)
        self.eng.bind_call_packed(points, offsets, list(max_n), layout=lay)
        self.eng.bind_packed_records(False, True)
        P = self.eng.bound_packed_records()
        self.out, self.out_off = P["nonground"], P["nonground_offsets"]

    def tick(self, stream):
        self.eng.run_bound_call(stream)


def capture(form, st):
    import torch
    with torch.cuda.stream(st):
        for _ in range(3):
            form.tick(st.cuda_stream)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            form.tick(st.cuda_stream)
    return g


def tick_leg(args, emit):
    import torch
    import pwpp_b200
    scans = kitti_scans()
    frames = [scans[k % len(scans)] for k in range(NF)]
    lens = np.array([len(a) for a in frames])
    max_n = lens + 2048
    off_h = np.concatenate([[0], np.cumsum(lens)])
    pts = torch.from_numpy(np.concatenate(frames + [np.zeros((1024, 4), np.float32)])).cuda()
    offsets = torch.tensor(off_h, dtype=torch.int64, device="cuda")
    for step, name in ((22, "velodyne22"), (16, "xyzi16")):
        lay = records_bench.layout(step)
        points = records_bench.make_records(pts, step).reshape(-1).contiguous()
        forms = {"today": Today(pwpp_b200, points, offsets, max_n, lay, step), "packed": Packed(pwpp_b200, points, offsets, max_n, lay, step)}
        st = torch.cuda.Stream()
        graphs = {k: capture(v, st) for k, v in forms.items()}
        for g in graphs.values():
            g.replay()
        torch.cuda.synchronize()
        a, b = forms["today"], forms["packed"]
        assert torch.equal(a.out_off, b.out_off), "the two forms' offsets differ"
        t = int(b.out_off[-1])
        assert torch.equal(a.out[:t], b.out[:t]), "the two forms' packed non-ground records differ"
        emit({"record": "check", "layout": name, "step": step, "frames": NF, "points": int(off_h[-1]), "nonground_records": t, "equal": True})
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for run in range(args.runs):
            times = {k: [] for k in forms}
            for _ in range(args.reps):
                for k, g in graphs.items():
                    ev[0].record(st)
                    with torch.cuda.stream(st):
                        g.replay()
                    ev[1].record(st)
                    ev[1].synchronize()
                    times[k].append(ev[0].elapsed_time(ev[1]) * 1e3)
            for k, v in times.items():
                emit({"record": "tick", "layout": name, "step": step, "form": k, "run": run, "frames": NF, "points": int(off_h[-1]),
                      "median_us": round(float(np.median(v)), 1), "p10_us": round(float(np.percentile(v, 10)), 1),
                      "p90_us": round(float(np.percentile(v, 90)), 1), "reps": args.reps})
        for f in forms.values():
            f.eng.close()
        del graphs, forms
        torch.cuda.synchronize()


def kernel_leg(args, emit):
    import torch
    import bench
    import synth
    import pwpp_b200
    F = 1024
    pts, offs = synth.make_batch(bench.SEED, 0, F, "kitti64", "cuda")
    offs_np = offs.numpy().astype(np.int64)
    sizes = np.diff(offs_np)
    npts = int(offs_np[-1])
    counts = torch.from_numpy(sizes.copy()).cuda()
    names = ("k_gather_record_parts", "k_gather_record_packed")
    for step in STEPS:
        buf = records_bench.make_records(pts, step).reshape(-1).contiguous()
        ptrs = [buf.data_ptr() + int(o) * step for o in offs_np[:-1]]
        e = pwpp_b200.Engine(device=0, num_streams=F)
        e.bind_call(ptrs, sizes.tolist(), [records_bench.layout(step)] * F, counts)
        e.bind_record_results()
        e.bind_packed_records()
        for _ in range(2):
            e.run_bound_call()
        e.synchronize()
        P = e.bound_packed_records()
        R = e.bound_record_results()
        cnt = R[3].cpu().numpy().astype(np.int64)
        for z, key in enumerate(("ground", "nonground")):
            po = P[key + "_offsets"].cpu().numpy()
            assert po.tolist() == np.concatenate([[0], np.cumsum(cnt[:, z])]).tolist(), f"step {step}: {key} offsets"
            cap = R[z].cpu().numpy()
            want = np.concatenate([cap[R[2][f]:R[2][f] + cnt[f, z] * step] for f in range(F)])
            assert np.array_equal(P[key].cpu().numpy().reshape(-1)[:len(want)], want), f"step {step}: packed {key}"
        times = {n: [] for n in names}
        for rnd in range(args.runs):
            got = kernel_times(e.run_bound_call, args.kreps, names, e.synchronize)
            for n in names:
                times[n] += got[n]
                emit({"record": "kernel", "kernel": n, "run": rnd, "frames": F, "points": npts, "listed": int(cnt.sum()), "step": step,
                      "traffic_bytes": int(cnt.sum()) * (2 * step + 4), "kernel_us_median": round(float(np.median(got[n])), 1),
                      "samples": len(got[n])})
        e.close()
        del buf
        torch.cuda.synchronize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--kreps", type=int, default=20)
    args = ap.parse_args()
    if args.out and os.path.exists(args.out):
        os.remove(args.out)

    def emit(r):
        records_bench.emit(r, args.out)
    emit(gpu_info())
    tick_leg(args, emit)
    kernel_leg(args, emit)
    emit(gpu_info())


if __name__ == "__main__":
    main()
