"""A/B of the class-L1 fit kernel (k_fit_warp with SOA staging, patches of 513–2048 points) against a parent build: bench.py's full line
for each build, alternated, with the outputs of a seeded sample compared bit for bit. Run on the GPU from the repository root
after build(), with the parent commit's tree built beside it:

  python tools/fit_l1_bench.py --parent DIR [--lib NAME=PATH ...] [--steps K] [--reps R] [--out FILE]

  --parent   repository tree of the parent commit, built (its bench.py runs from there, with its own library and drivers)
  --lib      extra builds of this tree's library (a libpwpp_b200.so built with other compile-time constants), run through
             PWPP_LIB; how the kernel's shape was chosen
  one JSON line per run (build, rep, ms_per_step, stage times of the default batch and of the recorded scans, streaming, dense1m,
  latency_us, the card and the SM clocks bench.py sampled inside its timed region), then one line per build comparing its
  --dump-outputs sample with the parent's
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_bench(tree, env_extra, steps, warmup, dump_dir):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup), "--no-cpu-baseline"]
    if dump_dir:
        cmd += ["--dump-outputs", dump_dir]
    env = dict(os.environ, **env_extra)
    p = subprocess.run(cmd, cwd=tree, env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
    if p.returncode != 0 or not lines:
        raise RuntimeError(f"bench.py in {tree} failed ({p.returncode}): {p.stderr[-2000:]}")
    return json.loads(lines[-1])


def record(build, rep, d):
    val = lambda k, f="value": (d.get(k) or {}).get(f)  # noqa: E731
    lat = d.get("latency_us") or {}
    return {"build": build, "rep": rep, "steps": d["steps"], "ms_per_step": d["ms_per_step"], "value": d["value"],
            "stage_ms": d["roofline"]["stage_ms"], "kitti_scans_ms": val("kitti_scans", "ms_per_step"),
            "kitti_scans_stage_ms": val("kitti_scans", "stage_ms"), "streaming": val("streaming"), "dense1m": val("dense1m"),
            "latency_us": {k: v for k, v in lat.items() if isinstance(v, (int, float))},
            "gpu": d.get("gpu"), "clocks": d.get("clocks")}


def same_outputs(a, b):
    names = sorted(f for f in os.listdir(a) if f.endswith(".npy"))
    if not names or names != sorted(f for f in os.listdir(b) if f.endswith(".npy")):
        return False
    return all(np.load(os.path.join(a, n)).tobytes() == np.load(os.path.join(b, n)).tobytes() for n in names)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True)
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    builds = [("parent", os.path.abspath(args.parent), {}), ("change", REPO, {})]
    for spec in args.lib:
        name, path = spec.split("=", 1)
        builds.append((name, REPO, {"PWPP_LIB": os.path.abspath(path)}))
    out = open(args.out, "a") if args.out else None

    def emit(r):
        line = json.dumps(r)
        print(line, flush=True)
        if out:
            out.write(line + "\n"); out.flush()

    with tempfile.TemporaryDirectory() as tmp:
        for rep in range(1, args.reps + 1):
            for name, tree, env in builds:
                dump = os.path.join(tmp, name) if rep == 1 else ""
                emit(record(name, rep, run_bench(tree, env, args.steps, args.warmup, dump)))
        for name, _, _ in builds[1:]:
            emit({"build": name, "dump_outputs_identical_to_parent": same_outputs(os.path.join(tmp, "parent"), os.path.join(tmp, name))})


if __name__ == "__main__":
    main()
