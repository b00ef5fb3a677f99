"""examples/pwpp_sequence.cpp in its several-streams form (DIR [DIR ...] [--frames-per-call K]) against the C-ABI stub
(tests/stub_pwpp_streams.c, labels by z; the stub's height of a stream is 1.723 + the frames it was given): call order, per-frame
counts, which lines carry a height, and that one directory without the flag still takes the single-stream path."""
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
SRC = os.path.join(REPO, "examples", "pwpp_sequence.cpp")


@pytest.fixture(scope="module")
def runner():
    build = os.path.join(HERE, "_build")
    os.makedirs(build, exist_ok=True)
    stub = os.path.join(build, "libpwpp_stub_streams.so")
    subprocess.check_call(["gcc", "-O1", "-shared", "-fPIC", "-I" + os.path.join(REPO, "include"), os.path.join(HERE, "stub_pwpp_streams.c"), "-o", stub])
    exe = os.path.join(build, "pwpp_sequence_stub_streams")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I" + os.path.join(REPO, "include"), SRC, "-o", exe, stub, "-Wl,-rpath," + build, "-lpthread"])
    return exe


def _dirs(tmp_path, kitti, lengths):
    """Directory d holds lengths[d] scans; scan t of directory d has 1000 * (d + 1) + 37 * t points of fixture scan (d + t) % 6."""
    dirs, scans = [], []
    for d, m in enumerate(lengths):
        p = tmp_path / f"seq{d}"
        p.mkdir()
        scans.append([])
        for t in range(m):
            a = np.ascontiguousarray(kitti[(d + t) % 6][:1000 * (d + 1) + 37 * t])
            a.tofile(p / f"{t:06d}.bin")
            scans[-1].append(a)
        dirs.append(str(p))
    return dirs, scans


def _run(exe, args):
    out = subprocess.run([exe, *args], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    return [l.split() for l in out.stdout.splitlines() if "points" in l.split()[1:3]], out.stdout.splitlines()[-1]


@pytest.mark.parametrize("k", [1, 2, 4])
def test_several_directories_time_major(tmp_path, kitti, runner, k):
    lengths = [3, 5, 2]
    dirs, scans = _dirs(tmp_path, kitti, lengths)
    lines, last = _run(runner, dirs + ["--frames-per-call", str(k)])
    want = []   # (stream, scan) in call order: K scans of every stream that still has scans, time-major
    for t0 in range(0, max(lengths), k):
        want += [(d, t) for t in range(t0, min(max(lengths), t0 + k)) for d in range(3) if t < lengths[d]]
    assert [(int(tok[0]), tok[1]) for tok in lines] == [(d, f"{t:06d}.bin") for d, t in want]
    for tok, (d, t) in zip(lines, want):
        a = scans[d][t]
        assert int(tok[3]) == len(a)
        assert int(tok[5]) == int((a[:, 2] < -1.5).sum()) and int(tok[5]) + int(tok[7]) == len(a)
    # a height is printed for the last frame of each stream in its call only: the stub's height is 1.723 + frames seen so far
    heights = {}
    for tok, (d, t) in zip(lines, want):
        if tok[11] != "-":
            heights[(d, t)] = float(tok[11])
    for d in range(3):
        ends = [min(t0 + k, lengths[d]) - 1 for t0 in range(0, lengths[d], k)]
        assert sorted(t for (dd, t) in heights if dd == d) == ends
        for t in ends:
            assert abs(heights[(d, t)] - (1.723 + t + 1)) < 1e-9
    assert f"{sum(lengths)} frames of 3 streams in {(max(lengths) + k - 1) // k} calls" in last


def test_frames_per_call_on_one_directory_and_the_single_stream_path(tmp_path, kitti, runner):
    dirs, scans = _dirs(tmp_path, kitti, [5])
    single, last = _run(runner, dirs)   # the drop-in class path: "<name> points ..." lines, as before
    assert "frames/s end to end" in last and "streams" not in last
    assert [tok[0] for tok in single] == [f"{t:06d}.bin" for t in range(5)]
    batched, last = _run(runner, dirs + ["--frames-per-call", "4"])
    assert "5 frames of 1 streams in 2 calls" in last
    assert [tok[1] for tok in batched] == [tok[0] for tok in single]
    for a, b in zip(single, batched):
        assert (a[2], a[4], a[6], a[8]) == (b[3], b[5], b[7], b[9])   # points, ground, non-ground, patches
    assert [tok[11] for tok in batched] == ["-", "-", "-", "5.7230", "6.7230"]


def test_a_library_without_the_stream_table(tmp_path, kitti):
    """Linked against a C-ABI without pwpp_estimate_host_streams (tests/stub_pwpp.c): the one-directory form runs as before,
    the several-streams form refuses with a message instead of failing to link."""
    build = os.path.join(HERE, "_build")
    os.makedirs(build, exist_ok=True)
    stub = os.path.join(build, "libpwpp_stub_nostreams.so")
    subprocess.check_call(["gcc", "-O1", "-shared", "-fPIC", "-I" + os.path.join(REPO, "include"), os.path.join(HERE, "stub_pwpp.c"), "-o", stub])
    exe = os.path.join(build, "pwpp_sequence_stub_nostreams")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I" + os.path.join(REPO, "include"), SRC, "-o", exe, stub, "-Wl,-rpath," + build, "-lpthread"])
    dirs, _ = _dirs(tmp_path, kitti, [3, 2])
    single, last = _run(exe, dirs[:1])
    assert [tok[0] for tok in single] == [f"{t:06d}.bin" for t in range(3)] and "3 frames" in last
    out = subprocess.run([exe, *dirs], capture_output=True, text=True, timeout=60)
    assert out.returncode == 1 and "no pwpp_estimate_host_streams" in out.stderr


def test_an_empty_directory_is_an_error(tmp_path, kitti, runner):
    dirs, _ = _dirs(tmp_path, kitti, [2])
    empty = tmp_path / "empty"; empty.mkdir()
    assert subprocess.run([runner, dirs[0], str(empty)], capture_output=True).returncode == 2
