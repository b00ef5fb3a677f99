"""What a packed bound call saves (pwpp_bind_call_packed + pwpp_bind_packed_xyz) against the scatter / compaction a pipeline needs
around a fixed-address bound call today. One JSON line per record on stdout and, with --out FILE, in FILE. Run on the GPU from
the repository root after build():

  python tools/bound_packed_bench.py [--out FILE] [--reps R] [--runs K]

  gpu     card name, power limit, maximum and current SM clock (nvidia-smi), read before and after the numbers in the same command
  tick    one tick of 64 KITTI-64 sensors whose scans arrive as one packed float32 (N, 4) tensor with device offsets, and whose
          consumer takes packed non-ground xyz, each form captured in one CUDA graph:
            today   a sync-free torch scatter of the packed batch into one fixed region per frame (searchsorted on the device
                    offsets), the counts from the offsets, a bound replay with capacity-layout non-ground xyz
                    (pwpp_bind_getter_results), then a sync-free torch compaction of those rows into one packed tensor;
            packed  a packed bind with packed non-ground xyz.
          Device time between CUDA events around one replay, median of --reps replays, the two forms alternated, --runs runs.
          Before timing, both forms' packed non-ground xyz and offsets are checked equal bit for bit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, "patchwork-plusplus_b200")
for p in (PKG, os.path.join(PKG, "lib"), REPO):
    if p not in sys.path:
        sys.path.insert(0, p)

NF = 64


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,driver_version"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, clk, cur, drv = [x.strip() for x in out[0].split(",")]
    return {"record": "gpu", "name": name, "power_limit": plim, "max_sm_clock": clk, "sm_clock": cur, "driver": drv}


def kitti_scans():
    d = os.path.join(REPO, "tests", "golden")
    names = sorted(f for f in os.listdir(d) if f.startswith("kitti_") and f.endswith(".npz"))
    return [np.ascontiguousarray(np.load(os.path.join(d, f))["xyzi_t"].T.astype(np.float32)) for f in names]


class Today:
    """Scatter -> bound call with capacity-layout xyz -> compaction, all device work with fixed shapes."""

    def __init__(self, pwpp_b200, points, offsets, max_n):
        import torch
        self.points, self.offsets = points, offsets
        self.N = points.shape[0]
        cap = np.concatenate([[0], np.cumsum(max_n)])
        self.rows = int(cap[-1])
        self.cap_off = torch.tensor(cap, dtype=torch.int64, device="cuda")
        self.regions = torch.zeros(self.rows + 1, 4, dtype=torch.float32, device="cuda")   # the last row takes what is not copied
        self.counts = torch.zeros(NF, dtype=torch.int64, device="cuda")
        self.ar_n = torch.arange(self.N, dtype=torch.int64, device="cuda")
        self.ar_r = torch.arange(self.rows, dtype=torch.int64, device="cuda")
        self.out = torch.zeros(self.rows + 1, 3, dtype=torch.float32, device="cuda")
        self.out_off = torch.zeros(NF + 1, dtype=torch.int64, device="cuda")
        self.eng = pwpp_b200.Engine(device=0, num_streams=NF)
        lay = pwpp_b200.layout_from_dtype(np.dtype({"names": ["x", "y", "z", "intensity"], "formats": ["<f4"] * 4, "offsets": [0, 4, 8, 12], "itemsize": 16}))
        base = self.regions.data_ptr()
        self.eng.bind_call([base + 16 * int(c) for c in cap[:-1]], list(max_n), [lay] * NF, self.counts)
        self.eng.bind_getter_results(False, True, False)
        G = self.eng.bound_getter_results()
        self.ng, self.cnt = G["nonground_xyz"], G["xyz_counts"]

    def tick(self, stream):
        import torch
        off = self.offsets
        f = torch.searchsorted(off[1:], self.ar_n, right=True).clamp_(max=NF - 1)   # frame of every packed record
        valid = self.ar_n < off[-1]
        dst = torch.where(valid, self.cap_off[f] + (self.ar_n - off[f]), self.rows)
        self.regions.index_copy_(0, dst, self.points)
        self.counts.copy_(off[1:] - off[:-1])
        self.eng.run_bound_call(stream)
        c = self.cnt[:, 1].to(torch.int64)
        self.out_off[1:] = torch.cumsum(c, 0)
        fr = torch.searchsorted(self.cap_off[1:], self.ar_r, right=True).clamp_(max=NF - 1)   # frame of every capacity row
        k = self.ar_r - self.cap_off[fr]
        keep = k < c[fr]
        dst = torch.where(keep, self.out_off[fr] + k, self.rows)
        self.out.index_copy_(0, dst, self.ng)


class Packed:
    def __init__(self, pwpp_b200, points, offsets, max_n):
        self.eng = pwpp_b200.Engine(device=0, num_streams=NF)
        self.eng.bind_call_packed(points, offsets, list(max_n))
        self.eng.bind_packed_xyz(False, True)
        P = self.eng.bound_packed_xyz()
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    import torch
    import pwpp_b200
    fh = open(args.out, "w") if args.out else None

    def emit(r):
        line = json.dumps(r)
        print(line, flush=True)
        if fh:
            fh.write(line + "\n")
    emit(gpu_info())
    scans = kitti_scans()
    frames = [scans[k % len(scans)] for k in range(NF)]
    lens = np.array([len(a) for a in frames])
    max_n = lens + 2048
    off_h = np.concatenate([[0], np.cumsum(lens)])
    points = torch.from_numpy(np.concatenate(frames + [np.zeros((1024, 4), np.float32)])).cuda()
    offsets = torch.tensor(off_h, dtype=torch.int64, device="cuda")
    forms = {"today": Today(pwpp_b200, points, offsets, max_n), "packed": Packed(pwpp_b200, points, offsets, max_n)}
    st = torch.cuda.Stream()
    graphs = {k: capture(v, st) for k, v in forms.items()}
    for g in graphs.values():
        g.replay()
    torch.cuda.synchronize()
    a, b = forms["today"], forms["packed"]
    assert torch.equal(a.out_off, b.out_off), "the two forms' offsets differ"
    t = int(b.out_off[-1])
    assert torch.equal(a.out[:t].view(torch.int32), b.out[:t].view(torch.int32)), "the two forms' packed non-ground xyz differ"
    emit({"record": "check", "frames": NF, "points": int(off_h[-1]), "nonground_rows": t, "equal": True})
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
            emit({"record": "tick", "form": k, "run": run, "frames": NF, "points": int(off_h[-1]), "median_us": float(np.median(v)),
                  "p10_us": float(np.percentile(v, 10)), "p90_us": float(np.percentile(v, 90)), "reps": args.reps})
    emit(gpu_info())
    if fh:
        fh.close()


if __name__ == "__main__":
    main()
